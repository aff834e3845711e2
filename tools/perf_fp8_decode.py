"""LLaMA-13B decode step with fp16 weights vs FP8 (e4m3) weights, measured in one process on one GPU.

Both models are built from one synthetic fp16 state dict (26 GB + 13 GB of weights, which fits an 80 GB card), the state dict is freed, and
each model's captured decode graph (the one generate_greedy_batch replays) is timed with CUDA events at B = 1 and B = 4 lock-step sequences,
alternating the two models window by window.  Prints ms per step, the weight bytes one step streams (from the tensor shapes), the
achieved GB/s and its share of the 3.35 TB/s HBM3 data-sheet bandwidth of an H100 SXM, then the prefill time at P = 182 for both formats and
the time of the FP8 model's dequantization kernels alone.

    python tools/perf_fp8_decode.py [--windows 10] [--steps 20]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from seedx_b200 import ops, synth  # noqa: E402
from seedx_b200.llm import LLAMA_13B, PROJECTIONS, LlamaForCausalLM  # noqa: E402

HBM_PEAK = 3.35e12     # bytes/s, H100 SXM data sheet
P = 182


def weight_bytes(m):
    """bytes of weights one decode step reads: every projection (+ its row scales), lm_head, the RMSNorm vectors"""
    nb = lambda t: t.numel() * t.element_size()  # noqa: E731
    total = nb(m.lm_head) + nb(m.norm)
    for L in m.layers:
        total += nb(L["ln1"]) + nb(L["ln2"])
        for k in PROJECTIONS:
            total += nb(L[k]) + (nb(L[k + "_s"]) if k + "_s" in L else 0)
    return total


def timed(fn, n=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10, help="alternating timing windows per model and batch size")
    ap.add_argument("--steps", type=int, default=20, help="graph replays per window")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi name, power.limit, clocks.max.sm: {smi}", flush=True)

    synth.set_device("cuda")
    sd = synth.llama_state_dict(LLAMA_13B)
    synth.set_device("cpu")
    max_len = P + 2 * args.steps + 64
    models = {}
    for fmt in ("fp16", "fp8_e4m3"):
        m = LlamaForCausalLM(LLAMA_13B, max_len=max_len, weight_format=fmt)
        m.load_state_dict(sd)
        models[fmt] = m
    del sd
    torch.cuda.empty_cache()
    print(f"weights resident: {torch.cuda.memory_allocated() / 1e9:.1f} GB; peak so far {torch.cuda.max_memory_allocated() / 1e9:.1f} GB", flush=True)
    wb = {fmt: weight_bytes(m) for fmt, m in models.items()}

    gen = torch.Generator().manual_seed(0)
    for B in (1, 4):
        ids = [torch.randint(3, 30000, (P,), generator=gen).tolist() for _ in range(B)]
        graphs, st0 = {}, {}
        for fmt, m in models.items():
            embs = [m.get_input_embeddings()(torch.tensor(i)).view(P, -1) for i in ids]
            m.generate_greedy_batch(ids, embs, max_new_tokens=2 * args.steps + 2, eos_id=2, suppress_eos=True)   # prefill + capture + pages
            graphs[fmt] = m._graphs[(B, 2, True)]
            st0[fmt] = m.state.clone()
            st0[fmt][:, 0] = P + 1          # every window restarts at the first decode position (its KV pages are reserved)
            st0[fmt][:, 1] = 0
            st0[fmt][:, 2] = 1
        ms = {fmt: [] for fmt in models}
        for w in range(args.windows + 1):
            for fmt, m in models.items():
                m.state.copy_(st0[fmt])
                t = timed(graphs[fmt].replay, args.steps)
                if w:                        # window 0 warms both graphs up
                    ms[fmt].append(t)
        for fmt in models:
            med = statistics.median(ms[fmt])
            print(f"B={B} {fmt:>8}: decode step {med:.3f} ms (median of {args.windows} windows x {args.steps} replays, spread "
                  f"{min(ms[fmt]):.3f}-{max(ms[fmt]):.3f}) | weights {wb[fmt] / 1e9:.3f} GB/step -> {wb[fmt] / med / 1e6:.0f} GB/s = "
                  f"{100 * wb[fmt] / med / 1e-3 / HBM_PEAK:.1f} % of 3.35 TB/s", flush=True)
        print(f"B={B} FP8 speed-up: {statistics.median(ms['fp16']) / statistics.median(ms['fp8_e4m3']):.2f}x", flush=True)

    emb = models["fp16"].get_input_embeddings()(torch.randint(3, 30000, (P,), generator=gen)).view(P, -1)
    pre = {fmt: [] for fmt in models}
    for w in range(6):
        for fmt, m in models.items():
            t = timed(lambda: m.prefill(emb, slot=0))
            if w:
                pre[fmt].append(t)
    m8 = models["fp8_e4m3"]

    def dequant_all():
        for L in m8.layers:
            for k in PROJECTIONS:
                ops.dequant_fp8(L[k], L[k + "_s"], m8._wscratch[:L[k].numel()].view(L[k].shape))
    dequant_all()
    dq = statistics.median(timed(dequant_all) for _ in range(5))
    for fmt in models:
        print(f"prefill P={P} {fmt:>8}: {statistics.median(pre[fmt]):.2f} ms (median of 5, spread {min(pre[fmt]):.2f}-{max(pre[fmt]):.2f})",
              flush=True)
    n8 = sum(L[k].numel() for L in m8.layers for k in PROJECTIONS)
    print(f"FP8 dequantization kernels of one prefill pass ({4 * len(m8.layers)} launches, {n8 / 1e9:.1f} GB read, {2 * n8 / 1e9:.1f} GB written): "
          f"{dq:.2f} ms", flush=True)


if __name__ == "__main__":
    main()
