"""Drop-in surface checked without a GPU: prompt layouts, grounding post-processing, the launcher for unmodified reference scripts, and a
static check that every keyword the reference's entry scripts pass to the factories / generate() / init_pipe() is a named parameter of the
replacement.  What these tests compare against was taken from the reference tree and is stored in tests/golden/dropin_reference.json
(tests/golden/make_dropin_golden.py regenerates it)."""
import hashlib
import inspect
import json
import os
import subprocess
import sys

import pytest
import torch

from seedx_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("SEEDX_REFERENCE", "/root/reference")
needs_ref = pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree not present")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "dropin_reference.json")))


def test_chat_prompt_layout_single_and_multi_turn():
    from seedx_b200 import demo
    tok = synth.SynthTokenizer()
    q = "What is in the image?"
    a_ids, a_mask = demo.image_prompt(tok, 3, q)
    b_ids, b_mask = demo.chat_prompt(tok, [q], views_per_image=[3])
    assert torch.equal(a_ids, b_ids) and torch.equal(a_mask, b_mask)          # one turn, one image == the eval_img2text layout
    assert int(a_mask.sum()) == 3 * 64
    # the layout of eval_img2text_seed_x_i.py:142-147 spelled out
    img = "".join("<img_{:05d}>".format(i) for i in range(64))
    text = "[INST] " + ("<patch>" + img + "</patch>") * 2 + "<img>" + img + "</img>" + q + " [/INST]\n"
    assert a_ids[0].tolist() == [tok.bos_token_id] + tok.encode(text)
    # two images (2 + 1 views), three turns, system message
    ids, mask = demo.chat_prompt(tok, ["q1", "a1", "q2"], views_per_image=[2, 1], system_message="sys")
    assert int(mask.sum()) == 3 * 64
    want = "sys\n[INST] " + "<patch>" + img + "</patch>" + "<img>" + img + "</img>" + "<img>" + img + "</img>" + "q1 [/INST]\na1\n[INST] q2 [/INST]\n"
    assert ids[0].tolist() == [tok.bos_token_id] + tok.encode(want)
    # masked rows are exactly the <img_k> ids, in order, once per view
    first = tok.tok2id["<img_00000>"]
    assert ids[0][mask[0]].tolist() == list(range(first, first + 64)) * 3
    ids_f, _ = demo.chat_prompt(tok, ["draw a cat"], force_image=True)
    assert ids_f[0, -1].item() == tok.tok2id["<img>"]
    with pytest.raises(ValueError):
        demo.chat_prompt(tok, ["q1", "a1"])


def test_extract_box_and_pixel_corners():
    from seedx_b200 import demo
    s = "The mask <box_start><loc-112><loc-56><loc-40><loc-20><box_end> and <box_start><loc-0><loc-223><loc-10><loc-5><box_end>."
    assert demo.extract_box(s) == [[112, 56, 40, 20], [0, 223, 10, 5]]
    assert demo.extract_box("no boxes here <loc-3>") is None
    # (x_center, y_center, w, h) in 224 bins on a 448 x 896 image
    assert demo.box_to_pixels([112, 56, 40, 20], 448, 896) == (184, 184, 264, 264)
    assert demo.box_to_pixels([0, 223, 10, 5], 448, 896) == (-10, 882, 10, 902)
    # the reference's extract_box (eval_img2text_seed_x_i.py) on the same strings
    for t, want in GOLDEN["extract_box"]:
        assert demo.extract_box(t) == want, t


def test_visualize_bbox_draws_the_rectangle(tmp_path):
    import numpy as np
    from PIL import Image
    from seedx_b200 import demo
    img = Image.new("RGB", (448, 224), (0, 0, 0))
    out = demo.visualize_bbox(img, [[112, 112, 56, 56]], str(tmp_path / "vis" / "g.png"))
    a = np.asarray(out)
    x1, y1, x2, y2 = demo.box_to_pixels([112, 112, 56, 56], 448, 224)
    assert (x1, y1, x2, y2) == (168, 84, 280, 140)
    assert tuple(a[y1, x1]) == (0, 255, 0) and tuple(a[y2, x2]) == (0, 255, 0) and tuple(a[(y1 + y2) // 2, (x1 + x2) // 2]) == (0, 0, 0)
    assert os.path.exists(tmp_path / "vis" / "g.png")


def test_launcher_runs_a_reference_style_script(tmp_path):
    """a script that begins like the reference's (top-level third-party imports, pyrootutils marker, sibling import, YAML `_target_`)
    runs unmodified through `python -m seedx_b200.run` even though hydra / omegaconf / pyrootutils / diffusers are not installed"""
    d = tmp_path / "proj" / "src" / "inference"
    os.makedirs(d)
    open(tmp_path / "proj" / ".project-root", "w").close()
    (d / "any_res.py").write_text("def process_anyres_image(*a):\n    return 'sibling import ok'\n")
    (d / "eval_demo.py").write_text(
        "import hydra\nimport torch\nimport os\nimport pyrootutils\nfrom omegaconf import OmegaConf\n"
        "from diffusers import AutoencoderKL, UNet2DConditionModel, EulerDiscreteScheduler\n"
        "from any_res import process_anyres_image\n"
        "root = pyrootutils.setup_root(__file__, indicator='.project-root', pythonpath=True)\n"
        "import sys\nassert __name__ == '__main__' and sys.argv[1:] == ['--flag']\n"
        "cfg = OmegaConf.load('configs/processer/qwen_448_transform.yaml')\n"
        "t = hydra.utils.instantiate(cfg)\n"
        "lc = OmegaConf.load('configs/clm_models/llm_seed_x_lora.yaml')\n"
        "print('OK', callable(t), process_anyres_image(), os.path.basename(str(root)), lc.peft_config.r, lc['vocab_size'])\n")
    r = subprocess.run([sys.executable, "-m", "seedx_b200.run", str(d / "eval_demo.py"), "--flag"], cwd=ROOT, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip().endswith("OK True sibling import ok proj 32 32330"), r.stdout


# ---- static call-surface check against the reference's own entry scripts ---------------------------------------------------------------
def _named_params(fn):
    return {p.name for p in inspect.signature(fn).parameters.values() if p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)}


def test_reference_scripts_only_use_keywords_the_replacement_names():
    from seedx_b200 import compat
    compat.install()
    from seedx_b200.adapter import SDXLAdapter, SDXLAdapterWithLatentImage
    from seedx_b200.agent import ContinuousLVLM
    from seedx_b200.sdxl import AutoencoderKL, EulerDiscreteScheduler, UNet2DConditionModel
    scripts = GOLDEN["entry_calls"]
    assert len(scripts) == 7
    seen = 0
    for name, script in sorted(scripts.items()):
        adapter_cls = SDXLAdapterWithLatentImage if script["edit"] else SDXLAdapter
        for c in script["calls"]:
            owner, attr = c["owner"], c["attr"]
            if attr == "generate" and owner == "agent_model":
                target = ContinuousLVLM.generate
            elif attr == "generate" and owner == "adapter":
                target = adapter_cls.generate
            elif attr == "init_pipe" and owner == "adapter":
                target = adapter_cls.init_pipe
            else:
                target = {"AutoencoderKL": AutoencoderKL, "UNet2DConditionModel": UNet2DConditionModel,
                          "EulerDiscreteScheduler": EulerDiscreteScheduler}[owner].from_pretrained
            missing = set(c["keywords"]) - _named_params(target)
            assert not missing, f"{name}:{c['line']} passes {sorted(missing)} which {target.__qualname__} does not name"
            seen += 1
    assert seen >= 20, seen


def test_import_block_of_every_reference_entry_script_executes_under_the_stand_ins():
    """the statements every reference entry script runs before touching a model — its top-level imports (incl. `from diffusers import …,
    Transformer2DModel` and the sibling `from any_res import …`) and `pyrootutils.setup_root` — execute against this repo exactly as
    `python -m seedx_b200.run <script>` would run them (compat.install() + script directory on sys.path); a missing name fails here, not on a GPU box"""
    def alias(n, a):
        return n + (" as " + a if a else "")
    blocks = {}
    for name, stmts in GOLDEN["entry_imports"].items():
        lines = []
        for st in stmts:
            if "import" in st:
                lines.append("import " + ", ".join(alias(n, a) for n, a in st["import"]))
            elif "from" in st:
                lines.append("from %s import %s" % (st["from"], ", ".join(alias(n, a) for n, a in st["names"])))
            else:
                lines.append("pyrootutils.setup_root(__file__, %s)" % ", ".join("%s=%r" % kv for kv in sorted(st["setup_root"].items())))
        assert len(lines) >= 7, name
        blocks[name] = "\n".join(lines)
    assert len(blocks) == 7
    code = r'''
import os, sys
sys.path.insert(0, %r)
from seedx_b200 import compat
compat.install()
sys.path.insert(0, os.path.join(%r, "src", "inference"))      # what seedx_b200.run does for the sibling import
for name, block in sorted(%r.items()):
    # __file__ of the script as the launcher sees it: the same relative location inside THIS repo
    ns = {"__name__": "not_main", "__file__": os.path.join(%r, "src", "inference", name)}
    exec(compile(block, name, "exec"), ns)
    import diffusers
    for n in ("AutoencoderKL", "UNet2DConditionModel", "EulerDiscreteScheduler"):
        assert ns[n] is getattr(diffusers, n)
    print("ok", name)
''' % (ROOT, ROOT, blocks, ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.count("ok eval_") == 7, r.stdout


def test_reference_yaml_targets_resolve_with_identical_keys():
    """every inference YAML of the reference has a twin here with the same `_target_`s and keys (values may differ only in comments):
    the parsed YAML, serialised canonically, hashes to the reference's"""
    import yaml
    from seedx_b200 import compat
    names = sorted(GOLDEN["yaml_digests"])
    assert len(names) == 13

    def targets(o, acc):
        if isinstance(o, dict):
            if "_target_" in o:
                acc.append(o["_target_"])
            for v in o.values():
                targets(v, acc)
        return acc

    for n in names:
        ours = yaml.safe_load(open(os.path.join(ROOT, "configs", n)))
        assert hashlib.sha256(json.dumps(ours, sort_keys=True).encode()).hexdigest() == GOLDEN["yaml_digests"][n], n
        for t in targets(ours, []):
            if t.startswith(("src.", "peft.")):
                compat.install()
                assert callable(compat._locate(t)), t


@needs_ref
def test_goldens_regenerate_bit_identically_from_the_reference(tmp_path):
    """tests/golden/*.pt ARE the outputs of the reference's own modules and dropin_reference.json holds facts read from the reference's files:
    running the generators again against the reference tree reproduces both exactly.  Needs the reference tree (SEEDX_REFERENCE)."""
    env = dict(os.environ, SEEDX_GOLDEN_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "golden", "make_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]

    def same(a, b, path):
        if torch.is_tensor(a):
            assert torch.is_tensor(b) and a.shape == b.shape and torch.equal(a, b), path
        elif isinstance(a, dict):
            assert a.keys() == b.keys(), path
            for k in a:
                same(a[k], b[k], f"{path}/{k}")
        elif isinstance(a, (list, tuple)):
            assert len(a) == len(b), path
            for i, (x, y) in enumerate(zip(a, b)):
                same(x, y, f"{path}[{i}]")
        else:
            assert a == b, path

    names = sorted(f for f in os.listdir(os.path.join(ROOT, "tests", "golden")) if f.endswith(".pt"))
    assert names == sorted(f for f in os.listdir(tmp_path) if f.endswith(".pt")) and len(names) == 8
    for f in names:
        same(torch.load(os.path.join(ROOT, "tests", "golden", f)), torch.load(tmp_path / f), f)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "golden", "make_dropin_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert json.load(open(tmp_path / "dropin_reference.json")) == GOLDEN


def test_anyres_preprocessing_equals_the_reference_on_random_sizes():
    """seedx_b200.preprocess vs the reference's own functions on 60 random image sizes and both transform modes: grid choice, tile order
    and patch positions exactly, pixel values bit for bit (sha256 of the float32 tensors the reference produced)"""
    code = r'''
import hashlib, json, sys, numpy as np, torch
from PIL import Image
sys.path.insert(0, "%s")
from seedx_b200 import preprocess as pp
golden = json.loads(%r)
def h(t):
    return hashlib.sha256(t.contiguous().float().numpy().tobytes()).hexdigest()
base = 448
grids = [[base * int(g[0]), base * int(g[2])] for g in ["1x1", "1x2", "1x3", "2x1", "3x1", "1x4", "4x1", "2x2"]]
rng = np.random.RandomState(7)
n = 0
for i in range(60):
    w, h_ = int(rng.randint(40, 2600)), int(rng.randint(40, 2600))
    g = golden[i]
    assert (g["w"], g["h"]) == (w, h_)
    img = Image.fromarray(rng.randint(0, 255, (h_, w, 3), dtype=np.uint8))
    use = grids if i %% 3 else grids[:1]
    v1, p1 = pp.process_anyres_image(img, pp.get_transform("clip", keep_ratio=False, image_size=base), use, base)
    assert list(v1.shape) == g["views_shape"] and p1.tolist() == g["patch_pos"] and h(v1) == g["views_sha256"], (w, h_)
    if i %% 10 == 0:
        k1 = pp.get_transform("clip", keep_ratio=True, image_size=base)(img)
        assert list(k1.shape) == g["keep_ratio_shape"] and h(k1) == g["keep_ratio_sha256"], (w, h_)
    n += 1
print("checked", n)
''' % (ROOT, json.dumps(GOLDEN["anyres"]))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.strip().endswith("checked 60")
