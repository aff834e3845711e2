"""FP8 (e4m3) UNet transformer projections against fp16 on one GPU, in one run:

1. the card: name, power limit, max SM clock;
2. seedx_gemm_fp8 against seedx_gemm_f16 at the transformer shapes of the i2i batch (8 samples: M = 8192 at C = 1280, M = 32768 at C = 640),
   CUDA events over rotating operand sets larger than L2, in TFLOP/s and as a share of the data-sheet dense peaks (989 fp16, 1979 FP8);
3. seedx_quant_rows_fp8: time and GB/s against 3.35 TB/s, and its share of one FP8 sample-forward (torch.profiler kernel times);
4. the UNet sample-forward at 8 samples replayed as a CUDA graph, fp16 and FP8 alternating, and the eps difference between them;
5. i2i images/s of SeedXEngine with the fp16 and the FP8 UNet on bench.py's seeded inputs (4 requests, 50 steps).

Usage: python tools/perf_fp8_unet.py [--out results.json] [--skip-engine]   (--out: also write every number as JSON to that path)"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from seedx_b200 import ops, synth  # noqa: E402
from seedx_b200.llm import quantize_fp8_rows  # noqa: E402

PEAK16, PEAK8, HBM = 989e12, 1979e12, 3.35e12
L2_BYTES = 50 * 2 ** 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def time_calls(fns, iters):
    """mean ms per call of fns[i % len(fns)] over `iters` calls (CUDA events), after one warm-up pass over every fn"""
    for f in fns:
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fns[i % len(fns)]()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gemm_rates(res):
    shapes = []
    for M, C in ((8192, 1280), (32768, 640)):
        shapes += [(f"GEGLU M={M}", M, 8 * C, C, True), (f"ff2 M={M}", M, C, 4 * C, False), (f"QKV M={M}", M, 3 * C, C, False),
                   (f"out M={M}", M, C, C, False)]
    rows = []
    for name, M, N, K, gated in shapes:
        set_bytes = (M * K + N * K) * 2
        n_sets = max(2, -(-2 * L2_BYTES // set_bytes))
        sets16, sets8 = [], []
        for i in range(n_sets):
            a = (torch.randn(M, K, device="cuda") * 0.5).half()
            w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
            qa, sa = ops.quant_rows_fp8(a)
            qw, sw = quantize_fp8_rows(w)
            sets16.append((a, w)), sets8.append((qa, qw, sa, sw))
        bias = torch.zeros(N, device="cuda")
        out = torch.empty((M, N // 2 if gated else N), device="cuda", dtype=torch.float16)
        kw = dict(bias=bias, act=ops.ACT_GELU, gated=True) if gated else dict(bias=bias)
        f16 = [lambda s=s: ops.gemm(s[0], s[1], out=out, **kw) for s in sets16]
        f8 = [lambda s=s: ops.gemm(s[0], s[1], out=out, a_scale=s[2], w_scale=s[3], **kw) for s in sets8]
        iters = max(20, int(2e13 / (2 * M * N * K)))
        t16, t8 = [], []
        for _ in range(3):                       # alternate the two, three rounds each
            t16.append(time_calls(f16, iters)), t8.append(time_calls(f8, iters))
        t16, t8 = min(t16), min(t8)
        fl = 2.0 * M * N * K
        r = dict(shape=name, M=M, N=N, K=K, fp16_ms=t16, fp8_ms=t8, fp16_tflops=fl / t16 / 1e9, fp8_tflops=fl / t8 / 1e9,
                 fp16_of_peak=fl / t16 / 1e-3 / PEAK16, fp8_of_peak=fl / t8 / 1e-3 / PEAK8, speedup=t16 / t8)
        rows.append(r)
        print(f"{name:14s} N={N:6d} K={K:5d}: fp16 {r['fp16_tflops']:6.0f} TFLOP/s ({100 * r['fp16_of_peak']:4.1f} % of 989)  "
              f"fp8 {r['fp8_tflops']:6.0f} TFLOP/s ({100 * r['fp8_of_peak']:4.1f} % of 1979)  x{r['speedup']:.2f}", flush=True)
        del sets16, sets8
        torch.cuda.empty_cache()
    res["gemm"] = rows
    qrows = []
    for M, C in ((8192, 1280), (8192, 5120), (32768, 640), (32768, 2560)):
        xs = [torch.randn(M, C, device="cuda").half() for _ in range(max(2, -(-2 * L2_BYTES // (M * C * 2))))]
        q, s = ops.quant_rows_fp8(xs[0])
        t = min(time_calls([lambda x=x: ops.quant_rows_fp8(x, q=q, scale=s) for x in xs], 200) for _ in range(3))
        b = M * C * 3 + M * 4
        qrows.append(dict(rows=M, cols=C, ms=t, gbs=b / t / 1e6, of_hbm=b / t / 1e-3 / HBM))
        print(f"quant_rows_fp8 [{M}, {C}]: {1e3 * t:7.1f} us, {b / t / 1e6:6.0f} GB/s ({100 * b / t / 1e-3 / HBM:4.1f} % of 3.35 TB/s)", flush=True)
    res["quant"] = qrows


def unet_forward(res):
    from seedx_b200.sdxl import SDXL_UNET, UNet2DConditionModel
    cfg = dict(SDXL_UNET)
    synth.set_device("cuda")
    try:
        sd = synth.unet_state_dict(cfg)
    finally:
        synth.set_device("cpu")
    m16, m8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    m16.load_state_dict(sd), m8.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    Be = 8
    ctx = synth.randn("pf8_ctx", (Be, 64, 2048)).cuda()
    te = synth.randn("pf8_te", (Be, 1280)).cuda()
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(Be, 1).cuda()
    x_nchw = synth.randn("pf8_x", (Be, 4, 128, 128)).cuda()
    x_in = ops.nchw_to_nhwc_f16(x_nchw, 8)
    t_dev = torch.full((Be,), 601.0, device="cuda")
    graphs, outs = {}, {}
    for name, m in (("fp16", m16), ("fp8", m8)):
        cond = m.prepare_cond(ctx, te, tid)
        m.forward_nhwc(x_in, t_dev, cond)                      # eager warm-up (workspaces, tickets, first launches)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                outs[name] = m.forward_nhwc(x_in, t_dev, cond)
        torch.cuda.current_stream().wait_stream(s)
        graphs[name] = (g, cond)
    times = {"fp16": [], "fp8": []}
    for _ in range(5):
        for name in ("fp16", "fp8"):
            times[name].append(time_calls([graphs[name][0].replay], 5))
    t16, t8 = min(times["fp16"]), min(times["fp8"])
    e = ((outs["fp8"].float() - outs["fp16"].float()).norm() / outs["fp16"].float().norm()).item()
    # quantiser share of one FP8 forward: kernel times from the profiler, eager
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m8.forward_nhwc(x_in, t_dev, graphs["fp8"][1])
        torch.cuda.synchronize()
    tot = qt = 0.0
    for ev in prof.key_averages():
        d = getattr(ev, "device_time_total", None)
        if d is None:
            d = ev.cuda_time_total
        tot += d
        if "quant_rows_fp8" in ev.key:
            qt += d
    res["unet"] = dict(samples=Be, fp16_ms=t16, fp8_ms=t8, speedup=t16 / t8, eps_rel_fp8_vs_fp16=e, quant_share_of_fp8_forward=qt / max(tot, 1e-9),
                       all_fp16_ms=times["fp16"], all_fp8_ms=times["fp8"])
    print(f"UNet sample-forward x{Be} (CUDA graph): fp16 {t16:.1f} ms, fp8 {t8:.1f} ms (x{t16 / t8:.3f}); eps rel fp8 vs fp16 {e:.3e}; "
          f"quantiser {100 * qt / max(tot, 1e-9):.1f} % of the FP8 forward's kernel time", flush=True)
    del m16, m8, graphs, outs
    torch.cuda.empty_cache()


def engine_rate(res, steps=50, reps=2):
    import bench
    from seedx_b200.engine import SeedXEngine
    W = bench.WORKLOADS["i2i"]
    B = W["default_batch"]
    out = {}
    for fmt in ("fp16", "fp8_e4m3"):
        eng = SeedXEngine(unet_weight_format=fmt)
        views = synth.image("bench_views_rank0", B * W["views"], 448).cuda()
        patch_pos = torch.tensor([[0.5, 0.5], [0.5, 0.5]] * B)
        g = torch.Generator().manual_seed(1234)
        text_ids = [torch.randint(3, eng.tok.base, (32,), generator=g).tolist() for _ in range(B)]
        noise = synth.randn("bench_latents_rank0", (B, 4, 128, 128)).half().float().cuda()
        run = lambda: eng.generate(views, patch_pos, text_ids, steps=steps, noise=noise, n_views=W["views"])   # noqa: E731
        u8 = run()
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(reps):
            u8 = run()
        torch.cuda.synchronize()
        dt = (time.time() - t0) / reps
        out[fmt] = dict(step_s=dt, images_per_s=B / dt, image=u8.float().cpu())
        print(f"i2i SeedXEngine, UNet {fmt}: {dt:.3f} s per step of {B} requests = {B / dt:.3f} images/s", flush=True)
        del eng
        torch.cuda.empty_cache()
    d = (out["fp8_e4m3"]["image"] - out["fp16"]["image"]).abs()
    res["engine"] = {k: {kk: vv for kk, vv in v.items() if kk != "image"} for k, v in out.items()}
    res["engine"]["image_mean_abs_diff_u8"] = float(d.mean())
    print(f"i2i images fp8 vs fp16: mean |diff| {float(d.mean()):.2f} of 255", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="write the results as JSON to this path (default: print only)")
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_fp8_unet.py measures on a GPU; none found")
    res = dict(card=card())
    print("card:", res["card"], flush=True)
    gemm_rates(res)
    unet_forward(res)
    if not args.skip_engine:
        engine_rate(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
        print("wrote", args.out)


if __name__ == "__main__":
    main()
