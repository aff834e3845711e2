"""Continuous batching of the denoising loop (serving.DenoiseBatcher) against the lock-step loop, at SDXL size (1024^2, synthetic weights),
4 slots, UNet formats fp16 and fp8_e4m3_conv, in one run:

1. the card: name, power limit, max SM clock;
2. per-step time at full occupancy: the batcher's graph (UNet forward over 4 slots + seedx_cfg_euler_slots) against DenoiseLoop at B = 4
   (UNet forward graph + seedx_cfg_euler_step), same process, alternated, after warm-up;
3. the slot step kernels (combine + advance) against seedx_cfg_euler_step at B = 4, CUDA events over many launches;
4. admission (resampler conditioning + prepare_cond over all slots + initialisation) and retirement (batch-1 VAE decode to uint8) costs;
5. a fixed arrival trace (16 requests, one every 7 step-times, step counts alternating 30 / 50) through the batcher and through FIFO
   lock-step batches of up to 4 requests of equal step count via adapter.generate: images/s and mean / p50 / p95 latency in ms, and the
   same trace in steps (a model without a GPU: every step costs 1, admission and retirement cost 0).

Clock for the trace: virtual.  Arrivals are placed at multiples of the measured full-occupancy step time; while work runs, the clock moves
by the measured (synchronised) wall time of that work; when nothing is runnable it jumps to the next arrival (no idle GPU time is spent).

Usage: python tools/perf_denoise_batcher.py [--out results.json] [--formats fp16,fp8_e4m3_conv] [--steps-only]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

N_REQ, EVERY, STEP_MIX, SLOTS = 16, 7, (30, 50), 4


def trace_requests():
    return [dict(arrive=EVERY * i, n=STEP_MIX[i % len(STEP_MIX)]) for i in range(N_REQ)]


def stats(lat):
    s = sorted(lat)
    pick = lambda q: s[min(len(s) - 1, int(round(q * (len(s) - 1))))]     # noqa: E731
    return dict(mean=statistics.fmean(s), p50=pick(0.5), p95=pick(0.95))


def steps_model():
    """the trace in steps: batcher (admit between steps into the lowest free slot) and FIFO lock-step batches (up to 4 requests with the
    head's step count, started when the previous batch ends)"""
    reqs = trace_requests()
    # batcher
    t, pending, live, fin, nxt = 0, [], [None] * SLOTS, {}, 0
    while len(fin) < len(reqs):
        while nxt < len(reqs) and reqs[nxt]["arrive"] <= t:
            pending.append(nxt)
            nxt += 1
        for s in range(SLOTS):
            if live[s] is None and pending:
                live[s] = [pending.pop(0), 0]
        if all(v is None for v in live):
            t = reqs[nxt]["arrive"]
            continue
        t += 1
        for s in range(SLOTS):
            if live[s] is not None:
                live[s][1] += 1
                if live[s][1] == reqs[live[s][0]]["n"]:
                    fin[live[s][0]] = t
                    live[s] = None
    cb = [fin[i] - r["arrive"] for i, r in enumerate(reqs)]
    cb_end = max(fin.values())
    # lock-step
    t, queue, nxt, fin = 0, [], 0, {}
    while len(fin) < len(reqs):
        while nxt < len(reqs) and reqs[nxt]["arrive"] <= t:
            queue.append(nxt)
            nxt += 1
        if not queue:
            t = reqs[nxt]["arrive"]
            continue
        n = reqs[queue[0]]["n"]
        batch = []
        while queue and len(batch) < SLOTS and reqs[queue[0]]["n"] == n:
            batch.append(queue.pop(0))
        t += n
        for i in batch:
            fin[i] = t
    ls = [fin[i] - r["arrive"] for i, r in enumerate(reqs)]
    return dict(batcher=dict(latency_steps=stats(cb), makespan_steps=cb_end), lockstep=dict(latency_steps=stats(ls), makespan_steps=max(fin.values())))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def build_adapter(fmt):
    from seedx_b200 import synth
    from seedx_b200.adapter import SDXLAdapter
    from seedx_b200.resampler_xl import ResamplerXLV2
    from seedx_b200.sdxl import SDXL_UNET, SDXL_VAE, AutoencoderKL, EulerDiscreteScheduler, UNet2DConditionModel
    from seedx_b200.vit import VisionTransformerWithAttnPool
    synth.set_device("cuda")
    try:
        # a 2-layer ViT: it only computes the (cached) negative features; the resampler, UNet and VAE are the SDXL-size ones
        vit = VisionTransformerWithAttnPool(image_size=448, patch_size=14, width=208, layers=2, heads=2, mlp_ratio=2.5, output_dim=4096)
        vit.load_state_dict(synth.vit_state_dict(width=208, layers=2, heads=2, mlp_width=520, output_dim=4096, n_queries=256, patch=14))
        rx = ResamplerXLV2(normalize=False, **synth.RESAMPLER_XL)
        rx.load_state_dict(synth.resampler_xl_state_dict(synth.RESAMPLER_XL))
        unet = UNet2DConditionModel(dict(SDXL_UNET), weight_format=fmt)
        unet.load_state_dict(synth.unet_state_dict(dict(SDXL_UNET)))
        vae = AutoencoderKL(dict(SDXL_VAE))
        vae.load_state_dict({k: v for k, v in synth.vae_state_dict(dict(SDXL_VAE)).items() if not k.startswith(("encoder.", "quant_conv"))})
        ad = SDXLAdapter(unet=unet, resampler=rx, vit_down=True)
        ad.init_pipe(vae=vae, scheduler=EulerDiscreteScheduler(), visual_encoder=vit, image_transform=None)
    finally:
        synth.set_device("cpu")
    return ad


def embeds(i):
    from seedx_b200 import synth
    return synth.randn(f"perf_batcher_feats_{i}", (1, 64, 4096)).cuda()


def sync_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def full_occupancy(ad, rounds=3, k=20):
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler
    from seedx_b200.serving import DenoiseBatcher
    b = DenoiseBatcher(ad, slots=SLOTS, max_steps=100, output_type="latent")
    for i in range(SLOTS):
        b.submit(embeds(i), num_inference_steps=100, seed=i, input_image_size=224)
    b.step()                                   # admits all 4, captures, first step
    loop = DenoiseLoop(ad.unet, EulerDiscreteScheduler(), SLOTS, (128, 128), 2, use_graph=True)
    p, n, pp, npool = ad.get_image_embeds(image_embeds=torch.cat([embeds(i) for i in range(SLOTS)]), image_size=224)
    tid = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]], device="cuda").repeat(2 * SLOTS, 1)
    loop.set_condition(torch.cat([n, p]), torch.cat([npool, pp]), tid)
    noise = torch.randn((SLOTS, 4, 128, 128), device="cuda")
    loop.run(noise, steps=2)                   # capture + warm-up
    for _ in range(2):
        b.step()
    cb, ls = [], []
    for _ in range(rounds):
        ms, _ = sync_time(lambda: [b.step() for _ in range(k)])
        cb.append(ms / k)
        ms, _ = sync_time(lambda: loop.run(noise, steps=k))
        ls.append(ms / k)
    while not b.idle():                         # finish the 4 requests (their slots are needed by nobody; keeps the batcher state clean)
        b.step()
    return dict(batcher_step_ms=cb, lockstep_step_ms=ls, batcher_step_ms_median=statistics.median(cb),
                lockstep_step_ms_median=statistics.median(ls), graph_kernels=b.graph_kernels, lockstep_graph_kernels=loop.graph_kernels + 1)


def slot_kernel_time(iters=50, chunks=8):
    from seedx_b200 import ops
    from seedx_b200.sdxl import EulerDiscreteScheduler
    S, h = SLOTS, 128
    x = torch.randn((S, 4, h, h), device="cuda")
    eps = torch.randn((2 * S, h, h, 4), device="cuda")
    u = torch.zeros((2 * S, h, h, 8), device="cuda", dtype=torch.float16)
    t = torch.zeros((2 * S,), device="cuda")
    sch = EulerDiscreteScheduler().set_timesteps(iters)
    sig = torch.tensor(sch.sigmas, device="cuda").repeat(S, 1)
    ts = torch.tensor(sch.timesteps, device="cuda").repeat(S, 1)
    sc = torch.tensor([[7.5, 1.5, sch.init_noise_sigma]], device="cuda").repeat(S, 1)
    st0 = torch.tensor([[0, iters]] * S, dtype=torch.int32, device="cuda")
    st = st0.clone()
    x0 = x.clone()
    res = {"slots": [], "lockstep": []}
    for c in range(chunks + 1):                 # chunk 0 is warm-up
        st.copy_(st0)
        x.copy_(x0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            ops.cfg_euler_slots(eps, x, u, t, st, sig, ts, sc, 2)
        e1.record()
        x.copy_(x0)
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        for i in range(iters):
            ops.cfg_euler_step(eps, x, u, 2, 7.5, 1.5, sch.sigmas[i], sch.sigmas[i + 1])
        e3.record()
        torch.cuda.synchronize()
        if c:
            res["slots"].append(e0.elapsed_time(e1) * 1e3 / iters)
            res["lockstep"].append(e2.elapsed_time(e3) * 1e3 / iters)
    return dict(slots_step_us=statistics.median(res["slots"]), cfg_euler_step_us=statistics.median(res["lockstep"]),
                note="slots = combine + advance launches; per launch pair / per launch, CUDA events around 50 back-to-back calls, median of 8")


def admission_retirement(ad, reps=3):
    from seedx_b200.serving import DenoiseBatcher
    b = DenoiseBatcher(ad, slots=SLOTS, max_steps=100, output_type="uint8")
    for i in range(SLOTS - 1):                  # three slots busy, one free: admission and retirement stall them
        b.submit(embeds(i), num_inference_steps=100, seed=i, input_image_size=224)
    b.step()
    adm, ret = [], []
    for r in range(reps + 1):
        b.submit(embeds(10 + r), num_inference_steps=1, seed=10 + r, input_image_size=224)
        ms_a, _ = sync_time(b._admit)
        b._replay()
        for v in b.live:
            if v is not None:
                v["done"] += 1
        slot = next(s for s, v in enumerate(b.live) if v is not None and v["n"] == 1)
        ms_r, _ = sync_time(lambda: b._retire(slot))
        if r:
            adm.append(ms_a)
            ret.append(ms_r)
    return dict(admission_ms=statistics.median(adm), retirement_ms=statistics.median(ret))


def run_trace(ad, step_ms):
    from seedx_b200.serving import DenoiseBatcher
    reqs = trace_requests()
    arrive = [r["arrive"] * step_ms for r in reqs]
    feats = [embeds(100 + i) for i in range(len(reqs))]
    # batcher
    b = DenoiseBatcher(ad, slots=SLOTS, max_steps=100, output_type="uint8")
    b.submit(feats[0], num_inference_steps=1, seed=0, input_image_size=224)      # warm-up: capture outside the timed trace
    b.run()
    now, nxt, fin, rid_of = 0.0, 0, {}, {}
    while len(fin) < len(reqs):
        while nxt < len(reqs) and arrive[nxt] <= now:
            rid_of[b.submit(feats[nxt], num_inference_steps=reqs[nxt]["n"], seed=nxt, input_image_size=224)] = nxt
            nxt += 1
        if b.idle():
            now = arrive[nxt]
            continue
        ms, done = sync_time(b.step)
        now += ms
        for rid, _ in done:
            fin[rid_of[rid]] = now
    cb = [fin[i] - arrive[i] for i in range(len(reqs))]
    cb_end = max(fin.values())
    # FIFO lock-step batches through adapter.generate
    for B in range(1, SLOTS + 1):               # warm-up: one DenoiseLoop (and its graph) per batch size
        ad.generate(image_embeds=torch.cat(feats[:B]), num_inference_steps=1, seed=0, input_image_size=224, output_type="uint8")
    now, queue, nxt, fin = 0.0, [], 0, {}
    while len(fin) < len(reqs):
        while nxt < len(reqs) and arrive[nxt] <= now:
            queue.append(nxt)
            nxt += 1
        if not queue:
            now = arrive[nxt]
            continue
        n = reqs[queue[0]]["n"]
        batch = []
        while queue and len(batch) < SLOTS and reqs[queue[0]]["n"] == n:
            batch.append(queue.pop(0))
        ms, _ = sync_time(lambda: ad.generate(image_embeds=torch.cat([feats[i] for i in batch]), num_inference_steps=n, seed=batch[0],
                                              input_image_size=224, output_type="uint8"))
        now += ms
        for i in batch:
            fin[i] = now
    ls = [fin[i] - arrive[i] for i in range(len(reqs))]
    return dict(batcher=dict(images_per_s=len(reqs) / (cb_end / 1e3), latency_ms=stats(cb), makespan_ms=cb_end),
                lockstep=dict(images_per_s=len(reqs) / (max(fin.values()) / 1e3), latency_ms=stats(ls), makespan_ms=max(fin.values())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--formats", default="fp16,fp8_e4m3_conv")
    ap.add_argument("--steps-only", action="store_true", help="print the trace model in steps and stop (no GPU needed)")
    a = ap.parse_args()
    res = dict(trace=dict(requests=N_REQ, every_steps=EVERY, step_mix=STEP_MIX, slots=SLOTS), steps_model=steps_model())
    print(json.dumps(res["steps_model"]))
    if not a.steps_only:
        if not torch.cuda.is_available():
            raise SystemExit("perf_denoise_batcher: no CUDA device (use --steps-only for the model in steps)")
        res["card"] = card()
        print("card:", res["card"], flush=True)
        res["slot_kernel"] = slot_kernel_time()
        print(json.dumps(res["slot_kernel"]), flush=True)
        for fmt in a.formats.split(","):
            ad = build_adapter(fmt)
            r = dict(full_occupancy=full_occupancy(ad))
            print(fmt, json.dumps(r["full_occupancy"]), flush=True)
            r.update(admission_retirement(ad))
            print(fmt, "admission / retirement ms:", r["admission_ms"], r["retirement_ms"], flush=True)
            r["trace"] = run_trace(ad, r["full_occupancy"]["batcher_step_ms_median"])
            print(fmt, json.dumps(r["trace"]), flush=True)
            res[fmt] = r
            del ad
            torch.cuda.empty_cache()
        res["card_end"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
