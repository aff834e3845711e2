"""FP8 (e4m3) UNet convolutions against fp16 on one GPU, in one run:

1. the card: name, power limit, max SM clock;
2. seedx_conv_fp8 against the fp16 implicit-GEMM conv at the 14 distinct shapes of the UNet's FP8 convs (8 samples, 128 x 128 latents), CUDA
   events, in TFLOP/s from the real channel counts (not the padded ones) and as a share of the data-sheet dense peaks (989 fp16, 1979 FP8);
   seedx_quant_images_fp8 on each conv input: time and GB/s (bytes of its two launches: x read twice, q written once) against 3.35 TB/s;
3. the UNet sample-forward at 8 samples replayed as a CUDA graph for fp16, fp8_e4m3 and fp8_e4m3_conv, alternating, and the eps difference of
   the FP8 formats against fp16;
4. the share of the quantisers in the fp8_e4m3_conv forward's kernel time (torch.profiler, a separate eager pass);
5. i2i images/s of SeedXEngine for the three UNet formats on bench.py's seeded inputs (4 requests, 50 steps).

Usage: python tools/perf_fp8_conv.py [--out results.json] [--skip-engine]   (--out: also write every number as JSON to that path)"""
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

PEAK16, PEAK8, HBM = 989e12, 1979e12, 3.35e12
FORMATS = ("fp16", "fp8_e4m3", "fp8_e4m3_conv")
# (h = w, C_in, C_out, how many of the 36 FP8 convs have this shape)
UNET_CONVS = [(128, 320, 320, 7), (64, 320, 640, 1), (64, 640, 640, 6), (32, 640, 1280, 1), (32, 1280, 1280, 10), (32, 2560, 1280, 2),
              (32, 1920, 1280, 1), (64, 1280, 1280, 1), (64, 1920, 640, 1), (64, 1280, 640, 1), (64, 960, 640, 1), (128, 640, 640, 1),
              (128, 960, 320, 1), (128, 640, 320, 2)]


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


def conv_rates(res, n=8):
    from seedx_b200.sdxl import conv_fp8, pack_conv
    rows = []
    for hw, c, cout, count in UNET_CONVS:
        xs = [torch.nn.functional.silu(torch.randn((n, hw, hw, c), device="cuda")).half() for _ in range(2)]
        w = torch.randn((cout, c, 3, 3), device="cuda") * (9 * c) ** -0.5
        w16 = pack_conv(w, "cuda")
        q8, s8 = conv_fp8(w16, c)
        bias = torch.zeros(cout, device="cuda")
        qx = [ops.quant_images_fp8(x) for x in xs]
        out = torch.empty((n, hw, hw, cout), device="cuda", dtype=torch.float16)
        f16 = [lambda x=x: ops.conv2d_nhwc(x, w16, out=out, bias=bias) for x in xs]
        f8 = [lambda a=a: ops.conv2d_nhwc(a[0], q8, out=out, bias=bias, a_scale=a[1], w_scale=s8) for a in qx]
        ws = ops.quant_images_fp8_ws(n, hw * hw * c, "cuda")
        fq = [lambda x=x, a=a: ops.quant_images_fp8(x, q=a[0], scale=a[1], ws=ws) for x, a in zip(xs, qx)]
        fl = 2.0 * n * hw * hw * cout * 9 * c
        iters = max(20, int(1e13 / fl))
        t16, t8, tq = [], [], []
        for _ in range(3):                       # alternate, three rounds each
            t16.append(time_calls(f16, iters)), t8.append(time_calls(f8, iters)), tq.append(time_calls(fq, 100))
        t16, t8, tq = min(t16), min(t8), min(tq)
        qbytes = n * hw * hw * c * 5
        r = dict(hw=hw, c_in=c, c_out=cout, convs=count, fp16_ms=t16, fp8_ms=t8, fp16_tflops=fl / t16 / 1e9, fp8_tflops=fl / t8 / 1e9,
                 fp16_of_peak=fl / t16 / 1e-3 / PEAK16, fp8_of_peak=fl / t8 / 1e-3 / PEAK8, speedup=t16 / t8, quant_us=1e3 * tq,
                 quant_gbs=qbytes / tq / 1e6, quant_of_hbm=qbytes / tq / 1e-3 / HBM, fp8_plus_quant_speedup=t16 / (t8 + tq))
        rows.append(r)
        print(f"conv {hw:3d}x{hw:<3d} {c:4d}->{cout:4d} (x{count}): fp16 {r['fp16_tflops']:5.0f} TFLOP/s ({100 * r['fp16_of_peak']:4.1f} % of 989)  "
              f"fp8 {r['fp8_tflops']:5.0f} TFLOP/s ({100 * r['fp8_of_peak']:4.1f} % of 1979)  x{r['speedup']:.2f};  quant {r['quant_us']:6.1f} us "
              f"{r['quant_gbs']:5.0f} GB/s ({100 * r['quant_of_hbm']:4.1f} % of 3.35 TB/s); fp8 + quant x{r['fp8_plus_quant_speedup']:.2f}", flush=True)
        del xs, qx, f16, f8, fq
        torch.cuda.empty_cache()
    res["conv"] = rows


def unet_forward(res):
    from seedx_b200.sdxl import SDXL_UNET, UNet2DConditionModel
    cfg = dict(SDXL_UNET)
    synth.set_device("cuda")
    try:
        sd = synth.unet_state_dict(cfg)
    finally:
        synth.set_device("cpu")
    models = {f: UNet2DConditionModel(cfg, weight_format=f) for f in FORMATS}
    for m in models.values():
        m.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    Be = 8
    ctx = synth.randn("pf8_ctx", (Be, 64, 2048)).cuda()
    te = synth.randn("pf8_te", (Be, 1280)).cuda()
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(Be, 1).cuda()
    x_in = ops.nchw_to_nhwc_f16(synth.randn("pf8_x", (Be, 4, 128, 128)).cuda(), 8)
    t_dev = torch.full((Be,), 601.0, device="cuda")
    graphs, outs = {}, {}
    for name, m in models.items():
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
    times = {f: [] for f in FORMATS}
    for _ in range(5):
        for name in FORMATS:
            times[name].append(time_calls([graphs[name][0].replay], 5))
    t = {f: min(v) for f, v in times.items()}
    err = {f: ((outs[f].float() - outs["fp16"].float()).norm() / outs["fp16"].float().norm()).item() for f in FORMATS[1:]}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        models["fp8_e4m3_conv"].forward_nhwc(x_in, t_dev, graphs["fp8_e4m3_conv"][1])
        torch.cuda.synchronize()
    tot = qi = qr = cv = 0.0
    for ev in prof.key_averages():
        d = getattr(ev, "device_time_total", None)
        if d is None:
            d = ev.cuda_time_total
        tot += d
        if "quant_images" in ev.key:
            qi += d
        elif "quant_rows_fp8" in ev.key:
            qr += d
        elif "gemm_tc_kernel" in ev.key and ("__nv_fp8_e4m3, true" in ev.key or "Lb1EEEv" in ev.key):   # the FP8 conv kernels (CONV8)
            cv += d
    tot = max(tot, 1e-9)
    res["unet"] = dict(samples=Be, ms={f: t[f] for f in FORMATS}, all_ms=times, speedup_vs_fp16={f: t["fp16"] / t[f] for f in FORMATS},
                       eps_rel_vs_fp16=err, quant_images_share=qi / tot, quant_rows_share=qr / tot, fp8_conv_share=cv / tot,
                       profiled_kernel_ms=tot / 1e3)
    print("UNet sample-forward x8 (CUDA graph): " + ", ".join(f"{f} {t[f]:.1f} ms (x{t['fp16'] / t[f]:.3f})" for f in FORMATS), flush=True)
    print("eps rel vs fp16: " + ", ".join(f"{f} {e:.3e}" for f, e in err.items()), flush=True)
    print(f"fp8_e4m3_conv forward kernel time (profiled, eager): per-image quantiser {100 * qi / tot:.1f} %, per-row quantiser "
          f"{100 * qr / tot:.1f} %, FP8 convs {100 * cv / tot:.1f} %", flush=True)
    del models, graphs, outs
    torch.cuda.empty_cache()


def engine_rate(res, steps=50, reps=2):
    import bench
    from seedx_b200.engine import SeedXEngine
    W = bench.WORKLOADS["i2i"]
    B = W["default_batch"]
    out = {}
    for fmt in FORMATS:
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
    res["engine"] = {k: {kk: vv for kk, vv in v.items() if kk != "image"} for k, v in out.items()}
    for f in FORMATS[1:]:
        d = float((out[f]["image"] - out["fp16"]["image"]).abs().mean())
        res["engine"][f]["image_mean_abs_diff_u8_vs_fp16"] = d
        print(f"i2i images {f} vs fp16: mean |diff| {d:.2f} of 255", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="write the results as JSON to this path (default: print only)")
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_fp8_conv.py measures on a GPU; none found")
    res = dict(card=card())
    print("card:", res["card"], flush=True)
    conv_rates(res)
    unet_forward(res)
    if not args.skip_engine:
        engine_rate(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)
        print("wrote", args.out)


if __name__ == "__main__":
    main()
