"""Generate tests/golden/dropin_reference.json from the reference tree (where it exists): the facts the drop-in tests compare against, stored as data.

* `entry_calls`: for every generate / init_pipe / from_pretrained call of the reference's src/inference/eval_*.py, the callee and the keyword names it passes
* `entry_imports`: the top-level imports of those scripts (module, [(name, alias)]) and whether they call pyrootutils.setup_root
* `yaml_digests`: sha256 of each inference YAML, parsed and re-serialised canonically (json, sorted keys)
* `extract_box`: the reference's extract_box on a few strings
* `anyres`: the reference's any-res preprocessing on 60 random image sizes: shapes, patch positions, sha256 of the float32 pixels

Run: python tests/golden/make_dropin_golden.py  (SEEDX_REFERENCE = the reference tree; SEEDX_GOLDEN_OUT = output directory)
"""
import ast
import glob
import hashlib
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("SEEDX_REFERENCE", "/root/reference")
YAMLS = ["visual_encoder/qwen_vitg_448.yaml", "processer/qwen_448_transform.yaml", "discrete_model/discrete_identity.yaml",
         "tokenizer/clm_llama_tokenizer_224loc_anyres.yaml", "clm_models/llm_seed_x.yaml", "clm_models/llm_seed_x_i.yaml",
         "clm_models/llm_seed_x_edit.yaml", "clm_models/llm_seed_x_lora.yaml", "clm_models/agent_seed_x.yaml", "clm_models/agent_seed_x_i.yaml",
         "clm_models/agent_seed_x_edit.yaml", "sdxl_adapter/sdxl_qwen_vit_resampler_l4_q64_pretrain_no_normalize.yaml",
         "sdxl_adapter/sdxl_qwen_vit_resampler_l4_q64_full_with_latent_image_pretrain_no_normalize.yaml"]
BOX_STRINGS = ["The mask <box_start><loc-112><loc-56><loc-40><loc-20><box_end> and <box_start><loc-0><loc-223><loc-10><loc-5><box_end>.",
               "none", "<box_start><loc-7><box_end><box_start><box_end>", "<box_start>a<loc-1>b<loc-22>c<box_end>"]


def yaml_digest(obj):
    return hashlib.sha256(json.dumps(obj, sort_keys=True).encode()).hexdigest()


def entry_scripts():
    scripts = sorted(glob.glob(os.path.join(REF, "src/inference/eval_*.py")))
    calls, imports = {}, {}
    for path in scripts:
        name = os.path.basename(path)
        src = open(path).read()
        tree = ast.parse(src)
        cs = []
        for node in ast.walk(tree):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute):
                owner = node.func.value.id if isinstance(node.func.value, ast.Name) else None
                if (node.func.attr, owner) in (("generate", "agent_model"), ("generate", "adapter"), ("init_pipe", "adapter")) or (
                        node.func.attr == "from_pretrained" and owner in ("AutoencoderKL", "UNet2DConditionModel", "EulerDiscreteScheduler")):
                    cs.append({"line": node.lineno, "owner": owner, "attr": node.func.attr,
                               "keywords": sorted(k.arg for k in node.keywords if k.arg is not None)})
        calls[name] = {"edit": "with_latent_image" in src, "calls": cs}
        im = []
        for node in tree.body:
            if isinstance(node, ast.Import):
                im.append({"import": [[a.name, a.asname] for a in node.names]})
            elif isinstance(node, ast.ImportFrom):
                im.append({"from": node.module, "names": [[a.name, a.asname] for a in node.names]})
            elif isinstance(node, ast.Expr) and isinstance(node.value, ast.Call) and getattr(node.value.func, "attr", "") == "setup_root":
                im.append({"setup_root": {k.arg: ast.literal_eval(k.value) for k in node.value.keywords if k.arg != "search_from"}})
        imports[name] = im
    return calls, imports


def ref_extract_box():
    path = os.path.join(REF, "src/inference/eval_img2text_seed_x_i.py")
    tree = ast.parse(open(path).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "extract_box")
    ns = {}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), {"re": re}, ns)
    return [[s, ns["extract_box"](s)] for s in BOX_STRINGS]


ANYRES = r'''
import hashlib, json, sys, numpy as np, torch
from PIL import Image
sys.path.insert(0, %r); sys.path.insert(0, %r)
from _ref_import import ref_module
ar, tr = ref_module("src.inference.any_res"), ref_module("src.processer.transforms")
def h(t):
    return hashlib.sha256(t.contiguous().float().numpy().tobytes()).hexdigest()
base = 448
grids = [[base * int(g[0]), base * int(g[2])] for g in ["1x1", "1x2", "1x3", "2x1", "3x1", "1x4", "4x1", "2x2"]]
rng = np.random.RandomState(7)
out = []
for i in range(60):
    w, h_ = int(rng.randint(40, 2600)), int(rng.randint(40, 2600))
    img = Image.fromarray(rng.randint(0, 255, (h_, w, 3), dtype=np.uint8))
    use = grids if i %% 3 else grids[:1]
    v0, p0 = ar.process_anyres_image(img, tr.get_transform("clip", keep_ratio=False, image_size=base), use, base)
    case = {"w": w, "h": h_, "views_shape": list(v0.shape), "views_sha256": h(v0), "patch_pos": p0.tolist()}
    if i %% 10 == 0:
        k0 = tr.get_transform("clip", keep_ratio=True, image_size=base)(img)
        case["keep_ratio_shape"], case["keep_ratio_sha256"] = list(k0.shape), h(k0)
    out.append(case)
print(json.dumps(out))
''' % (ROOT, HERE)


def main():
    calls, imports = entry_scripts()
    import yaml
    anyres = subprocess.run([sys.executable, "-c", ANYRES], capture_output=True, text=True, check=True, cwd=ROOT).stdout
    g = {"entry_calls": calls, "entry_imports": imports,
         "yaml_digests": {n: yaml_digest(yaml.safe_load(open(os.path.join(REF, "configs", n)))) for n in YAMLS},
         "extract_box": ref_extract_box(), "anyres": json.loads(anyres.strip().splitlines()[-1])}
    out = os.path.join(os.environ.get("SEEDX_GOLDEN_OUT", HERE), "dropin_reference.json")
    with open(out, "w") as f:
        json.dump(g, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
