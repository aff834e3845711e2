"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a GPU and exports every entry point that include/seedx.h
declares; the product path refuses to run without CUDA (no CPU fallback); host-side builder / scheduler / tokenizer logic."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "seedx.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(seedx_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from seedx_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared_symbols()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert _lib.lib().seedx_abi_version() == 2
    # nothing is launched by importing / loading the library: checked in a fresh interpreter, so that GPU tests run earlier in this process
    # (whose launches the counter rightly includes) do not matter
    probe = "import sys; sys.path.insert(0, sys.argv[1]); from seedx_b200 import _lib; _lib.lib(); print(_lib.launch_count())"
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", probe, ROOT], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "0", r.stdout


def test_no_cpu_fallback():
    from seedx_b200 import _lib, ops
    a = torch.zeros((8, 8), dtype=torch.float16)
    with pytest.raises(_lib.SeedxError):
        ops.gemm(a, a)
    with pytest.raises(_lib.SeedxError):
        ops.layernorm(a.float(), None, None, 1e-5)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "seed-x_b200")
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            src = open(os.path.join(pkg, f)).read()
            assert "import oracle" not in src and "from oracle" not in src, f


def test_instantiate_targets_and_overrides():
    from seedx_b200 import compat
    compat.install()
    import hydra
    from omegaconf import OmegaConf
    cfg = OmegaConf.load(os.path.join(ROOT, "configs", "clm_models", "agent_seed_x_i.yaml"))
    assert cfg.input_resampler.embed_dim == 5120 and cfg._target_.endswith("ContinuousLVLM.from_pretrained")
    tr = hydra.utils.instantiate(OmegaConf.load(os.path.join(ROOT, "configs", "processer", "qwen_448_transform.yaml")))
    assert tr.size == 448 and tr.keep_ratio is False
    r = hydra.utils.instantiate(cfg.input_resampler)          # nested _target_ -> hyper-parameter holder
    assert (r.grid_size, r.embed_dim, r.num_heads, r.kv_dim) == (8, 5120, 32, 4096)
    d = hydra.utils.instantiate(OmegaConf.load(os.path.join(ROOT, "configs", "discrete_model", "discrete_identity.yaml")))
    x = torch.ones(2)
    assert d.encode_image_embeds(x) is x
    # every YAML's _target_ resolves to an importable callable
    for dirpath, _, files in os.walk(os.path.join(ROOT, "configs")):
        for f in files:
            c = OmegaConf.load(os.path.join(dirpath, f))
            if "transformers." in c["_target_"]:
                continue
            assert callable(compat._locate(c["_target_"])), f


def test_scheduler_tables_match_oracle():
    from oracle import sdxl as osd
    from seedx_b200.sdxl import EulerDiscreteScheduler
    for n in (50, 30, 8):
        a, b = EulerDiscreteScheduler().set_timesteps(n), osd.Euler().set_timesteps(n)
        assert a.timesteps == [float(t) for t in b.timesteps.tolist()]
        assert max(abs(x - float(y)) for x, y in zip(a.sigmas, b.sigmas)) < 2e-5
        assert abs(a.init_noise_sigma - b.init_noise_sigma) < 2e-5


def test_synth_tokenizer_and_prompt_layout():
    from seedx_b200 import demo, synth
    tok = synth.SynthTokenizer()
    assert tok.vocab == 32330
    ids = tok.encode("<img><img_00000><img_00063></img>x")
    assert ids[0] == tok.tok2id["<img>"] and ids[2] == tok.tok2id["<img_00063>"] and ids[3] == tok.tok2id["</img>"] and 3 <= ids[4] < tok.base
    input_ids, mask = demo.image_prompt(tok, 3, "what is this?", force_image=True)
    assert mask.sum().item() == 3 * 64 and input_ids[0, 0].item() == tok.bos_token_id and input_ids[0, -1].item() == tok.tok2id["<img>"]
    assert tok.decode(tok.encode("<patch></patch>")) == "<patch></patch>"


def test_synth_is_deterministic():
    from seedx_b200 import synth
    a, b = synth.randn("x.y", (4, 5), 0.3), synth.randn("x.y", (4, 5), 0.3)
    assert torch.equal(a, b) and not torch.equal(a, synth.randn("x.z", (4, 5), 0.3))
    assert torch.equal(a, a.half().float())      # fp16-representable


def test_scheduler_known_answers():
    """Published constants of the Stable-Diffusion scaled-linear schedule (beta 0.00085..0.012, 1000 steps): sigma_min = 0.0292,
    sigma_max = 14.6146 (k-diffusion / diffusers defaults); 'leading' spacing with steps_offset 1 visits t = 981, 961, ..., 1 at 50 steps
    (SURVEY.md B.2).  Pins the scheduler tables independently of the in-repo oracle."""
    from seedx_b200.sdxl import EulerDiscreteScheduler
    s = EulerDiscreteScheduler()
    assert abs(s._sig[0] - 0.0292) < 5e-5 and abs(s._sig[-1] - 14.6146) < 5e-5
    a = s.set_timesteps(50)
    assert a.timesteps == [float(t) for t in range(981, 0, -20)] and len(a.sigmas) == 51 and a.sigmas[-1] == 0.0
    assert all(x > y for x, y in zip(a.sigmas, a.sigmas[1:]))
    assert abs(a.init_noise_sigma - (a.sigmas[0] ** 2 + 1) ** 0.5) < 1e-12 and abs(a.sigmas[0] - s._sig[981]) < 1e-12


def test_integration_md_ctypes_stub_mirrors_the_gemm_struct():
    """INTEGRATION.md shows the ctypes binding a reference maintainer would add; the library reads the whole seedx_gemm_args, so the stub must carry
    every field at the offset of the real binding (which the tests above pin against include/seedx.h)."""
    import ctypes as C
    import re
    from seedx_b200._lib import GemmArgs as Real
    src = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    m = re.search(r"class GemmArgs\(C.Structure\):.*?\n(    _fields_ = \[.*?\]\n)", src, re.S)
    assert m, "INTEGRATION.md no longer shows the GemmArgs stub"
    ns = {"C": C}
    exec("class GemmArgs(C.Structure):\n" + m.group(1), ns)
    stub = ns["GemmArgs"]
    assert C.sizeof(stub) == C.sizeof(Real)
    assert [n for n, _ in stub._fields_] == [n for n, _ in Real._fields_]
    for n, _ in stub._fields_:
        assert getattr(stub, n).offset == getattr(Real, n).offset, n
