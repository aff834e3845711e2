"""The kernels of the LLaMA token loop (csrc/llm_decode.cu): decode attention, RoPE + KV-cache prefill, the logits processor with greedy argmax,
and the embedding / scatter / hidden-state row copies, each against a float64 reference written here, at 13B width (40 heads of 128) and at
the tiny test model's 2 heads.  Every test also runs the CPU test double (tests/fake_ops.py) on copies of the same inputs: the CPU suite trusts
it to behave like the kernels.

Inputs come from seeded CPU generators; q/k/v values sit on a 1/64 grid with at most 11 significant bits, so fp16, fp32 and float64 hold them
exactly and every difference measured below comes from the kernel's arithmetic.
"""
import pytest
import torch

import fake_ops
from fp16_ulp import ulp16
from seedx_b200 import synth
from seedx_b200.llm import AutoImageTokenGenerationProcessor

pytestmark = pytest.mark.gpu

HD = 128
SCALE = float(torch.tensor(HD ** -0.5, dtype=torch.float32))            # the fp32 softmax scale ops.decode_attention passes
INV_FREQ = 1.0 / (10000.0 ** (torch.arange(0, HD, 2).float() / HD))    # fp32, built as LlamaForCausalLM builds it
SENT = 1234.0   # fills every cache row a launch must leave alone: exact in fp16 and far outside the |x| < 32 drawn here

# Attention output against float64 softmax(q K^T scale) V over the kernel's own cache rows, as max |error| / max |v|; "measured" is the
# worst over all cases on an H100 80GB HBM3 (SXM, 700 W power limit).  The kernel's error is fp32 rounding only: the fp32 RoPE of q and the
# 128-term fp32 dot product (~2^-24 sqrt(128) |q||k| scale, a few 1e-8 of these unit-variance scores), __expf (~2^-22 relative, plus
# |s - max| 2^-24 from scaling its argument by log2 e) and up to 2048/16 = 128 sequential fp32 p*v accumulations per half-warp before the
# 16-group merge, which stay near 2^-24 relative because the p are positive.
ATTN_TOL = 1.5e-7        # measured 4.6e-8
# Scores spread over ~150 (test_decode_attention_online_softmax_rescale): the argument error of __expf, |s - max| 2^-24 ~ 9e-6 relative for
# the farthest weights that still count, dominates.
RESCALE_TOL = 4e-6       # measured 1.3e-6
# The test double's fp32 einsum sums the 128 products and the softmax in a different order: each is within ~ATTN_TOL of float64, and the
# two fp32 RoPEs of q (cosf vs the CPU's cos) differ by an ulp of the angle's cosine here and there.
# In the prefill -> decode chain the two caches also differ by one fp16 ulp in a few elements (see CHAIN_TOL).
FAKE_ATTN_TOL = 2e-6     # measured 5.6e-7 (one decode step), 1.05e-6 (chain)
# ... and with scores spread over ~150 the fp32 rounding of each score, ~|s| 2^-24 absolute, moves the weights by as much relative.
FAKE_RESCALE_TOL = 8e-6  # measured 2.4e-6
# The prefill -> decode chain compares against float64 attention over fp16(RoPE64(k)), the correctly rounded cache.  Where the exact
# rotation lies within its fp32 error of an fp16 rounding boundary, the kernel's cache element lands one ulp away (307 of 2.9e6 elements
# here), which moves a score by scale |q_i| ulp16(k_i); that dominates the fp32 rounding above.
CHAIN_TOL = 3e-6         # measured 9.5e-7


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def grid(shape, seed, scale=1.0):
    """~N(0, scale^2) rounded to multiples of 1/64, |n/64| < 32: exactly representable in fp16 (11 significant bits), fp32 and float64"""
    return (torch.round(torch.randn(shape, generator=gen(seed)) * (64 * scale)).clamp(-2047, 2047) / 64).float()


def rope64(x, pos):
    """float64 rotate-half RoPE of x [..., H, 128] at integer positions pos [...].  The angle is the fp32 product pos * inv_freq that the
    kernels and HF form, so the test measures the kernel's rotation and not the rounding of the angle."""
    ang = (pos.float()[..., None] * INV_FREQ.to(pos.device)).double()
    c, s = ang.cos()[..., None, :], ang.sin()[..., None, :]
    x = x.double()
    x0, x1 = x[..., : HD // 2], x[..., HD // 2:]
    return torch.cat([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1)


def rope_slack(x):
    """bound on the fp32 error of a rotation computed in fp32 with cosf/sinf (2 ulp each): (|x0| + |x1|) 2^-21"""
    x = x.double().cpu()
    return torch.cat([x[..., : HD // 2].abs() + x[..., HD // 2:].abs()] * 2, dim=-1) * 2.0 ** -21


def check_rope(got, x, pos):
    """got: fp16 RoPE of x at pos, computed once in fp32 and rounded to fp16.  It must be within 1 fp16 ulp of fp16(RoPE64(x)): the fp32
    result is within half an ulp plus rope_slack(x), and the slack only matters where the rotation cancels to within ~2^-12 of its inputs,
    where the fp16 ulp is that small too.  Returns (worst difference in ulps, number of elements that differ)."""
    r16 = rope64(x, pos).half().double().cpu()
    d = (got.double().cpu() - r16).abs()
    u = ulp16(r16)
    assert (d <= u + rope_slack(x)).all(), f"RoPE off by {(d / u).max().item():.2f} fp16 ulps"
    return (d / u).max().item(), int((d != 0).sum())


def same_rope(a, b, x):
    """two fp16 roundings of the same fp32-computed rotation (kernel and test double): each within half an ulp plus rope_slack of the exact
    value, so within 1 ulp plus twice the slack of each other"""
    a, b = a.double().cpu(), b.double().cpu()
    return bool(((a - b).abs() <= ulp16(a) + 2 * rope_slack(x.reshape(-1, HD)).reshape(a.shape)).all())


def attn64(q, K, V, pos):
    """float64 decode attention for one slot: q fp32 [H*128] (rotated here), K/V [pos+1, H*128] -> [H*128]"""
    H = q.numel() // HD
    qr = rope64(q.view(H, HD), torch.tensor(pos, device=q.device))
    K, V = K.double().view(-1, H, HD), V.double().view(-1, H, HD)
    p = (torch.einsum("hd,thd->ht", qr, K) * SCALE).softmax(-1)
    return torch.einsum("ht,thd->hd", p, V).reshape(-1)


def rel_v(o, ref, V):
    """max |o - ref| / max |v|.  A non-finite output (a fully masked row gives 0/0) counts as an infinite error, so it cannot drop out of a
    running max() the way a NaN would."""
    e = ((o.double() - ref.to(o.device)).abs().max() / V.double().abs().max()).item()
    return e if bool(torch.isfinite(o).all()) and e == e else float("inf")


class Layout:
    """The cache of B sequences as one flat fp16 pool [rows, D], contiguous (slot b owns rows b*L .. b*L + L-1) or paged (pages of `page` rows
    handed out shuffled and interleaved across the slots, two pages owned by nobody)."""

    def __init__(self, lens, D, page, seed, L=None):
        self.B, self.D, self.page = len(lens), D, page
        if page:
            need = [(n + page - 1) // page for n in lens]
            self.n_pages = sum(need) + 2
            perm = iter(torch.randperm(self.n_pages, generator=gen(seed)).tolist())
            self.pt = torch.zeros((self.B, max(need)), dtype=torch.int32)
            for j in range(max(need)):
                for b in range(self.B):
                    if j < need[b]:
                        self.pt[b, j] = next(perm)
            self.rows = self.n_pages * page
        else:
            self.L = L or max(lens) + 16     # rows past every sequence's end must keep the sentinel too
            self.rows = self.B * self.L
        self.k = torch.full((self.rows, D), SENT, dtype=torch.float16, device="cuda")
        self.v = torch.full((self.rows, D), SENT, dtype=torch.float16, device="cuda")

    def row(self, b, t):
        t = torch.as_tensor(t, dtype=torch.long)
        if self.page:
            return self.pt[b].long()[t // self.page] * self.page + t % self.page
        return b * self.L + t

    def kv_args(self):
        if self.page:
            return (self.k.view(self.n_pages, self.page, self.D), self.v.view(self.n_pages, self.page, self.D),
                    dict(page_table=self.pt.cuda(), page_size=self.page))
        return self.k.view(self.B, self.L, self.D), self.v.view(self.B, self.L, self.D), {}

    def fake_args(self):
        """the same pool on the CPU for the test double, which takes paged caches only: a contiguous cache is one page per slot"""
        if self.page:
            return self.k.cpu().view(self.n_pages, self.page, self.D), self.v.cpu().view(self.n_pages, self.page, self.D), self.pt, self.page
        return self.k.cpu().view(self.B, self.L, self.D), self.v.cpu().view(self.B, self.L, self.D), torch.arange(self.B, dtype=torch.int32)[:, None], self.L


def untouched(after, before, written):
    keep = torch.ones(after.shape[0], dtype=torch.bool, device=after.device)
    keep[written.to(after.device)] = False
    return torch.equal(after[keep], before[keep])


# ------------------------------------------------------------------------------------------------------------------------------------------
# decode_attention
# ------------------------------------------------------------------------------------------------------------------------------------------
def _decode_inputs(H, lens, seed):
    B, D = len(lens), H * HD
    qkv = grid((B, 3 * D), seed)
    hist = [(grid((n - 1, D), seed + 1 + b).half(), grid((n - 1, D), seed + 101 + b).half()) for b, n in enumerate(lens)]
    state = torch.zeros((B, 4), dtype=torch.int32)
    state[:, 0] = torch.tensor(lens)
    return qkv, hist, state


def _decode_run(H, lens, qkv, hist, state, page, seed):
    """fills the history rows 0..len-2 of every slot, launches decode_attention once; returns (out, layout, pools before the launch)"""
    lay = Layout(lens, H * HD, page, seed)
    for b, (hk, hv) in enumerate(hist):
        r = lay.row(b, torch.arange(lens[b] - 1)).cuda()
        lay.k[r], lay.v[r] = hk.cuda(), hv.cuda()
    before = (lay.k.clone(), lay.v.clone())
    kc, vc, kw = lay.kv_args()
    out = torch.empty((len(lens), H * HD), device="cuda")
    from seedx_b200 import ops
    ops.decode_attention(qkv.cuda(), state.cuda(), INV_FREQ.cuda(), kc, vc, out, H, HD, **kw)
    torch.cuda.synchronize()
    return out, lay, before


@pytest.mark.parametrize("H,lens", [
    (40, [2048]),                                    # one slot at max_len
    (40, [1, 64, 373, 2048]),                        # pos 0 (15 of 16 half-warps own no token), one full 64-token unroll, any-res, max_len
    (40, [1, 63, 64, 65, 127, 129, 373, 501]),       # around the 64-token unroll stride, and the any-res lengths 373 and 373 + 128
    (2, [255]),                                      # the tiny test model: the last 64-token walk ends one short of a full group
])
def test_decode_attention(H, lens, record_property):
    """One decode step per slot, slots of different lengths in one launch, over a contiguous cache and over 16- and 64-token pages handed out
    shuffled: the new K row (RoPE, 1 fp16 ulp) and V row (exact) land at the slot's position and nowhere else, the output matches float64
    attention over the kernel's own cache rows, the three layouts give the same bits, and a slot alone gives the bits it gives in company."""
    B, D = len(lens), H * HD
    pos = [n - 1 for n in lens]
    qkv, hist, state = _decode_inputs(H, lens, 1000 + H + B)
    outs, rows_k, rows_v = {}, {}, {}
    worst_ulp = worst_attn = worst_fake = 0.0
    k_diff = 0
    for page in (0, 16, 64):
        out, lay, (k0, v0) = _decode_run(H, lens, qkv, hist, state, page, 7 + page)
        written = torch.stack([lay.row(b, pos[b]) for b in range(B)])
        assert untouched(lay.k, k0, written) and untouched(lay.v, v0, written), "a cache row other than the slot's position changed"
        for b in range(B):
            w = int(written[b])
            u, n = check_rope(lay.k[w].view(H, HD), qkv[b, D:2 * D].view(H, HD), torch.tensor(pos[b]))
            worst_ulp, k_diff = max(worst_ulp, u), k_diff + n
            assert torch.equal(lay.v[w].cpu(), qkv[b, 2 * D:].half())
            r = lay.row(b, torch.arange(lens[b])).cuda()
            ref = attn64(qkv[b, :D].cuda(), lay.k[r], lay.v[r], pos[b])
            worst_attn = max(worst_attn, rel_v(out[b], ref, lay.v[r]))
        outs[page], rows_k[page], rows_v[page] = out, lay.k[written.cuda()], lay.v[written.cuda()]
        if page == 16:
            fk, fv, fpt, fps = lay.fake_args()
            fk0, fv0 = k0.cpu().view_as(fk), v0.cpu().view_as(fv)
            fo = torch.empty((B, D))
            fake_ops.decode_attention(qkv.clone(), state.clone(), INV_FREQ, fk0, fv0, fo, H, HD, page_table=fpt, page_size=fps)
            assert torch.equal(fv0, fv)
            assert untouched(fk0.view(-1, D), fk.view(-1, D), written)
            for b in range(B):
                w = int(written[b])
                check_rope(fk0.view(-1, D)[w].view(H, HD), qkv[b, D:2 * D].view(H, HD), torch.tensor(pos[b]))
                assert same_rope(fk.view(-1, D)[w], fk0.view(-1, D)[w], qkv[b, D:2 * D])
                worst_fake = max(worst_fake, rel_v(fo[b], out[b].cpu().double(), fv.view(-1, D)[lay.row(b, torch.arange(lens[b]))]))
    record_property("k_row_ulps", worst_ulp)
    record_property("k_row_elements_off_by_one_ulp", k_diff)
    record_property("attn_err_vs_f64", worst_attn)
    record_property("fake_attn_err_vs_kernel", worst_fake)
    assert worst_attn <= ATTN_TOL, worst_attn
    assert worst_fake <= FAKE_ATTN_TOL, worst_fake
    for page in (16, 64):       # kv_row only changes addresses: same arithmetic in the same order
        assert torch.equal(outs[page], outs[0]) and torch.equal(rows_k[page], rows_k[0]) and torch.equal(rows_v[page], rows_v[0])
    if B > 1:
        for b in range(B):
            alone, _, _ = _decode_run(H, [lens[b]], qkv[b:b + 1], hist[b:b + 1], state[b:b + 1], 0, 7)
            assert torch.equal(alone[0], outs[0][b]), f"slot {b} alone differs from slot {b} in a batch"


@pytest.mark.parametrize("growth", [1.5, 16.0])
def test_decode_attention_online_softmax_rescale(growth, record_property):
    """Keys aligned with q whose magnitude rises with position: every 64-token block raises the running maximum of the online softmax, at
    growth 16 by a factor of e^4.5 to e^9 per block, and the scores of the first tokens fall more than 104 below the maximum, so their fp32
    weights underflow to exactly 0 against the final maximum."""
    H, lens = 40, [1000, 2048]
    B, D = len(lens), H * HD
    qkv, _, state = _decode_inputs(H, lens, 77)
    hist = []
    for b, n in enumerate(lens):
        qd = torch.sign(rope64(qkv[b, :D].view(H, HD), torch.tensor(n - 1))).float().reshape(D)
        ramp = growth * torch.arange(n - 1).float()[:, None] / n
        k = qd[None, :] * ramp + grid((n - 1, D), 300 + b, 0.25)
        hist.append((k.half(), grid((n - 1, D), 400 + b).half()))
    out, lay, (k0, v0) = _decode_run(H, lens, qkv, hist, state, 0, 5)
    out64, _, _ = _decode_run(H, lens, qkv, hist, state, 64, 5)
    assert torch.isfinite(out).all() and torch.equal(out, out64)
    # the test double over CPU copies of the same cache
    fk, fv, fpt, fps = lay.fake_args()
    fk0, fv0 = k0.cpu().view_as(fk), v0.cpu().view_as(fv)
    fo = torch.empty((B, D))
    fake_ops.decode_attention(qkv.clone(), state.clone(), INV_FREQ, fk0, fv0, fo, H, HD, page_table=fpt, page_size=fps)
    assert torch.equal(fv0, fv)
    worst = worst_fake = 0.0
    for b, n in enumerate(lens):
        r = lay.row(b, torch.arange(n)).cuda()
        if growth > 10:
            qr = rope64(qkv[b, :D].view(H, HD).cuda(), torch.tensor(n - 1, device="cuda"))
            s = torch.einsum("hd,thd->ht", qr, lay.k[r].double().view(n, H, HD)) * SCALE
            assert ((s.max(-1).values - s[:, 0]) > 104).all(), "the first token's weight should underflow in fp32"
        worst = max(worst, rel_v(out[b], attn64(qkv[b, :D].cuda(), lay.k[r], lay.v[r], n - 1), lay.v[r]))
        w = int(lay.row(b, n - 1))
        assert same_rope(fk.view(-1, D)[w], fk0.view(-1, D)[w], qkv[b, D:2 * D])
        worst_fake = max(worst_fake, rel_v(fo[b], out[b].cpu().double(), fv.view(-1, D)[r.cpu()]))
    record_property("attn_err_vs_f64", worst)
    record_property("fake_attn_err_vs_kernel", worst_fake)
    assert worst <= RESCALE_TOL, worst
    assert worst_fake <= FAKE_RESCALE_TOL, worst_fake


def test_prefill_then_decode_chain(record_property):
    """rope_kv_prefill of P tokens into shuffled 16-token pages, then 5 decode steps advancing state[0]: every step's output against float64
    attention over the whole sequence, with the cache taken as the correctly rounded fp16 RoPE of every k."""
    from seedx_b200 import ops
    H, P, steps = 40, [174, 373], 5
    B, D = len(P), H * HD
    lay = Layout([p + steps for p in P], D, 16, 11)
    kc, vc, kw = lay.kv_args()
    fk, fv, fpt, _ = lay.fake_args()                 # the test double runs the same chain over CPU copies of the pools
    inv = INV_FREQ.cuda()
    ks, vs = [], []
    for b in range(B):
        x = grid((P[b], 3 * D), 500 + b)
        ops.rope_kv_prefill(x.half().cuda(), 0, H, HD, inv, kc, vc, page_table_row=kw["page_table"][b], page_size=16)
        fake_ops.rope_kv_prefill(x.half(), 0, H, HD, INV_FREQ, fk, fv, page_table_row=fpt[b], page_size=16)
        ks.append(x[:, D:2 * D])
        vs.append(x[:, 2 * D:])
    state = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
    state[:, 0] = torch.tensor(P, dtype=torch.int32)
    out, fo = torch.empty((B, D), device="cuda"), torch.empty((B, D))
    worst = worst_fake = 0.0
    k_diff = 0
    for step in range(steps):
        state[:, 0] += 1
        qkv = grid((B, 3 * D), 600 + step)
        ops.decode_attention(qkv.cuda(), state, inv, kc, vc, out, H, HD, **kw)
        fake_ops.decode_attention(qkv.clone(), state.cpu(), INV_FREQ, fk, fv, fo, H, HD, page_table=fpt, page_size=16)
        assert torch.isfinite(out).all(), f"step {step}: non-finite attention output"
        for b in range(B):
            ks[b] = torch.cat([ks[b], qkv[b:b + 1, D:2 * D]])
            vs[b] = torch.cat([vs[b], qkv[b:b + 1, 2 * D:]])
            n = P[b] + step + 1
            K = rope64(ks[b].view(n, H, HD).cuda(), torch.arange(n, device="cuda")).half().view(n, D)
            ref = attn64(qkv[b, :D].cuda(), K, vs[b].cuda(), n - 1)
            e = rel_v(out[b], ref, vs[b])
            assert e <= CHAIN_TOL, (step, b, e)
            worst = max(worst, e)
            worst_fake = max(worst_fake, rel_v(fo[b], out[b].cpu().double(), vs[b]))
            if step == steps - 1:
                rows = lay.row(b, torch.arange(n))
                k_diff += int((lay.k[rows.cuda()] != K).sum())
                assert same_rope(lay.k[rows.cuda()], fk.view(-1, D)[rows], ks[b])
    assert torch.equal(fv.view(-1, D), lay.v.cpu())
    assert untouched(fk.view(-1, D), lay.k.cpu(), torch.cat([lay.row(b, torch.arange(P[b] + steps)) for b in range(B)]))
    record_property("chain_err_vs_f64", worst)
    record_property("chain_k_elements_off_by_one_ulp", k_diff)
    record_property("fake_attn_err_vs_kernel", worst_fake)
    assert worst_fake <= FAKE_ATTN_TOL, worst_fake


# ------------------------------------------------------------------------------------------------------------------------------------------
# rope_kv_prefill
# ------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("H", [2, 40])
@pytest.mark.parametrize("pos0", [0, 131])          # 131: a later chunk of a chunked prefill, starting mid-page
@pytest.mark.parametrize("T", [1, 7, 174, 373])
def test_rope_kv_prefill(T, pos0, H, paged, record_property):
    """q and k of the fp16 [T, 3D] block are rotated in place within 1 fp16 ulp of float64 RoPE, v is untouched, the rotated k and the v land
    in the cache rows of positions pos0 .. pos0+T-1 (through shuffled 16-token pages when paged) and every other row keeps its sentinel.
    The row decode_attention writes for the same k at the same position agrees within 1 fp16 ulp."""
    from seedx_b200 import ops
    D = H * HD
    x = grid((T, 3 * D), 40 * T + H + pos0).half()
    qkv = x.cuda()
    lay = Layout([pos0 + T], D, 16 if paged else 0, T + pos0)
    k0, v0 = lay.k.clone(), lay.v.clone()
    kc, vc, kw = lay.kv_args()
    ops.rope_kv_prefill(qkv, pos0, H, HD, INV_FREQ.cuda(), kc, vc, page_table_row=kw["page_table"][0] if paged else None, page_size=16 if paged else 0)
    torch.cuda.synchronize()
    pos = torch.arange(pos0, pos0 + T)
    uq, nq = check_rope(qkv[:, :D].view(T, H, HD), x[:, :D].view(T, H, HD), pos)
    uk, nk = check_rope(qkv[:, D:2 * D].view(T, H, HD), x[:, D:2 * D].view(T, H, HD), pos)
    record_property("q_ulps", uq)
    record_property("k_ulps", uk)
    assert torch.equal(qkv[:, 2 * D:].cpu(), x[:, 2 * D:])
    rows = lay.row(0, pos).cuda()
    assert torch.equal(lay.k[rows], qkv[:, D:2 * D]) and torch.equal(lay.v[rows], qkv[:, 2 * D:])
    assert untouched(lay.k, k0, rows) and untouched(lay.v, v0, rows)

    # the test double on CPU copies: q/k held to the same float64 bound, the same rows written, v exact
    fk, fv, fpt, fps = lay.fake_args()
    fk0, fv0 = k0.cpu().view_as(fk), v0.cpu().view_as(fv)
    fx = x.clone()
    fake_ops.rope_kv_prefill(fx, pos0, H, HD, INV_FREQ, fk0, fv0, page_table_row=fpt[0], page_size=fps)
    check_rope(fx[:, :D].view(T, H, HD), x[:, :D].view(T, H, HD), pos)
    check_rope(fx[:, D:2 * D].view(T, H, HD), x[:, D:2 * D].view(T, H, HD), pos)
    assert same_rope(fx[:, :2 * D], qkv[:, :2 * D], x[:, :2 * D])
    assert torch.equal(fx[:, 2 * D:], x[:, 2 * D:]) and torch.equal(fv0, fv)
    assert untouched(fk0.view(-1, D), fk.view(-1, D), rows.cpu())
    assert same_rope(fk0.view(-1, D)[rows.cpu()], fk.view(-1, D)[rows.cpu()], x[:, D:2 * D])

    # decode_attention writing the same k at the same positions (one slot per position, zero-filled contiguous caches)
    sel = sorted(set([0, 1, T // 3, T // 2, T - 2, T - 1]) & set(range(T)))
    p = [pos0 + t for t in sel]
    dq = torch.zeros((len(sel), 3 * D))
    dq[:, D:2 * D] = x[sel, D:2 * D].float()
    st = torch.zeros((len(sel), 4), dtype=torch.int32)
    st[:, 0] = torch.tensor(p, dtype=torch.int32) + 1
    dk = torch.zeros((len(sel), max(p) + 1, D), dtype=torch.float16, device="cuda")
    dv = torch.zeros_like(dk)
    ops.decode_attention(dq.cuda(), st.cuda(), INV_FREQ.cuda(), dk, dv, torch.empty((len(sel), D), device="cuda"), H, HD)
    dec = torch.stack([dk[j, p[j]] for j in range(len(sel))]).double()
    pre = qkv[sel, D:2 * D].double()
    record_property("prefill_vs_decode_k_elements_differing", int((dec != pre).sum()))
    assert ((dec - pre).abs() <= ulp16(pre)).all()


# ------------------------------------------------------------------------------------------------------------------------------------------
# logits_argmax
# ------------------------------------------------------------------------------------------------------------------------------------------
VOCAB = 32330
MAX_LEN = 40
TOK = synth.SynthTokenizer(vocab=VOCAB)
PROC = AutoImageTokenGenerationProcessor(TOK)                 # <img>, <img_00000> .. <img_00063>, </img>
IMG = PROC.img_ids_list
EOS = TOK.eos_token_id


def greedy64(logits, seq, state, img_ids, eos_id, suppress_eos):
    """the device step restated on host copies: AutoImageTokenGenerationProcessor.__call__ on the slot's ids (in float64), EOS at -inf under
    suppress_eos unless the span forces the id, torch.argmax; a slot that is parked (state[1] != 0) or full (state[0] == max_len) keeps its
    sequence and state"""
    seq, state = seq.clone(), state.clone()
    for b in range(logits.shape[0]):
        n = int(state[b, 0])
        scores = logits[b:b + 1].double().clone()
        forced = img_ids is not None and int(seq[b, n - 1]) in IMG[:-1]
        if img_ids is not None:
            PROC(seq[b:b + 1, :n], scores)
        if suppress_eos and not forced:
            scores[0, eos_id] = float("-inf")
        nxt = int(torch.argmax(scores[0]))
        if n < seq.shape[1] and int(state[b, 1]) == 0:
            seq[b, n] = nxt
            state[b, 0] = n + 1
            state[b, 2] += 1
            if eos_id is not None and nxt == eos_id and not suppress_eos:
                state[b, 1] = state[b, 2]
    return seq, state


def _slots(seed, n_slots=8):
    g = gen(seed)
    logits = torch.randn((n_slots, VOCAB), generator=g) * 3
    seq = torch.randint(3, TOK.base, (n_slots, MAX_LEN), generator=g, dtype=torch.int32)
    state = torch.zeros((n_slots, 4), dtype=torch.int32)
    state[:, 0] = torch.randint(2, MAX_LEN - 4, (n_slots,), generator=g, dtype=torch.int32)
    state[:, 2] = torch.randint(0, 9, (n_slots,), generator=g, dtype=torch.int32)
    return logits, seq, state


def _cases_with_span():
    logits, seq, state = _slots(1)
    last = lambda b, tok: seq.__setitem__((b, int(state[b, 0]) - 1), tok)   # noqa: E731
    # 0: plain argmax
    # 1: equal maxima in different threads and warps: 1023 (thread 1023, warp 31) beats 1024 (thread 0, second pass) and later ones
    logits[1, [1023, 1024, 5 * 1024 + 17, 31000]] = 50.0
    # 2: equal maxima in the strided walk of one thread (thread 3): the lowest, 2051, wins
    logits[2, [3 + 7 * 1024, 3 + 2 * 1024, 3 + 20 * 1024]] = 50.0
    # 3-5: the span forces the next id whatever the logits say (the processor writes max + 10, which must not round back to max)
    logits[3:6, 7] = 100.0
    last(3, IMG[0])                                  # <img> -> <img_00000>
    last(4, IMG[18])                                 # <img_00017> -> <img_00018>
    last(5, IMG[64])                                 # <img_00063> -> </img>
    # 6: after </img> nothing is forced; with every logit negative the 0.0 written into img_ids[1:] wins, lowest id first
    logits[6] = -(logits[6].abs() + 0.1)
    last(6, IMG[65])
    # 7: EOS chosen without suppression: state[1] = 1-based index of the EOS among the generated tokens
    logits[7, EOS] = 60.0
    return logits, seq, state


def _cases_suppress():
    logits, seq, state = _slots(2)
    logits[0, EOS], logits[0, 777] = 60.0, 40.0          # EOS suppressed: the runner-up
    logits[1, EOS], state[1, 1] = 60.0, 3               # parked
    state[2, 0] = MAX_LEN                               # full
    logits[3, [9000, 12000]], logits[3, 5] = float("nan"), 1e30      # NaN ranks above every number, the lowest NaN first (torch.argmax)
    logits[4, EOS] = 60.0
    seq[4, int(state[4, 0]) - 1] = IMG[63]              # <img_00062> -> <img_00063>, EOS or not
    logits[5, [100, 20000]] = float("inf")              # +inf ties: lowest index
    logits[6, EOS], state[6, 1] = 60.0, 1
    logits[7, 31999] = 80.0                             # the last warp's last pass
    return logits, seq, state


def _cases_no_span():
    logits, seq, state = _slots(3)
    logits[0] = float("-inf")                           # nothing is finite: id 0, as torch.argmax
    logits[1] = float("nan")                            # nothing is a number: id 0
    seq[2, int(state[2, 0]) - 1] = IMG[0]               # <img> without a span list forces nothing
    logits[3, 4096] = float("nan")
    logits[3, 64] = float("inf")
    logits[4, [0, 1024, 2048]] = 90.0
    return logits, seq, state


@pytest.mark.parametrize("name,build,img,eos,suppress", [
    ("span", _cases_with_span, True, EOS, False),
    ("suppress_eos", _cases_suppress, True, EOS, True),
    ("no_span", _cases_no_span, False, None, False),
])
def test_logits_argmax(name, build, img, eos, suppress):
    """8 slots over the 32330-id vocabulary per launch; the appended ids and all four state fields are exact against the logits processor
    (seedx_b200.llm.AutoImageTokenGenerationProcessor) followed by torch.argmax, and so is the test double."""
    from seedx_b200 import ops
    logits, seq, state = build()
    want_seq, want_state = greedy64(logits, seq, state, IMG if img else None, eos, suppress)
    img_ids = torch.tensor(IMG, dtype=torch.int32) if img else None
    dl, ds, dst = logits.cuda(), seq.cuda(), state.cuda()
    ops.logits_argmax(dl, img_ids.cuda() if img else None, ds, dst, eos, suppress)
    assert torch.equal(ds.cpu(), want_seq), (ds.cpu()[want_seq != ds.cpu()], want_seq[want_seq != ds.cpu()])
    assert torch.equal(dst.cpu(), want_state)
    fs, fst = seq.clone(), state.clone()
    fake_ops.logits_argmax(logits.clone(), img_ids, fs, fst, eos, suppress)
    assert torch.equal(fs, want_seq) and torch.equal(fst, want_state)
    if name == "suppress_eos":      # parked and full slots do not move
        for b in (1, 2, 6):
            assert torch.equal(ds.cpu()[b], seq[b]) and torch.equal(dst.cpu()[b], state[b])


# ------------------------------------------------------------------------------------------------------------------------------------------
# embed_rows, scatter_rows, store_hidden: copies, bit-exact
# ------------------------------------------------------------------------------------------------------------------------------------------
def test_embed_rows():
    from seedx_b200 import ops
    V, D = 3000, 5120
    table = (torch.randn((V, D), generator=gen(1)) * 2).half()
    ids = torch.randint(0, V, (37,), generator=gen(2), dtype=torch.int32)
    ids[0], ids[-1] = 0, V - 1
    out = torch.full((37, D), SENT, device="cuda")
    ops.embed_rows(table.cuda(), out, ids=ids.cuda())
    want = table[ids.long()].float()
    assert torch.equal(out.cpu(), want)
    assert torch.equal(fake_ops.embed_rows(table, torch.empty((37, D)), ids=ids), want)
    # device-resident sequences: row b embeds seq[b, state[b,0] - 1], seq a view whose row stride (96) exceeds its length (64)
    B = 5
    full = torch.randint(0, V, (B, 96), generator=gen(3), dtype=torch.int32)
    seq = full[:, :64]
    state = torch.zeros((B, 4), dtype=torch.int32)
    state[:, 0] = torch.tensor([1, 17, 63, 64, 40], dtype=torch.int32)
    dfull = full.cuda()
    out = torch.full((B, D), SENT, device="cuda")
    ops.embed_rows(table.cuda(), out, state=state.cuda(), seq=dfull[:, :64])
    want = table[torch.stack([seq[b, int(state[b, 0]) - 1] for b in range(B)]).long()].float()
    assert torch.equal(out.cpu(), want)
    assert torch.equal(fake_ops.embed_rows(table, torch.empty((B, D)), state=state, seq=seq), want)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("gather", [False, True])
def test_scatter_rows(dtype, gather):
    from seedx_b200 import ops
    D, R = 5120, 40
    src = (torch.randn((9, D), generator=gen(4)) * 3).to(dtype)
    idx = torch.tensor([7, 2, 31, 5, 39, 0], dtype=torch.int32)          # scattered, out of order
    src_idx = torch.tensor([8, 0, 3, 3, 6, 1], dtype=torch.int32) if gather else None
    dst0 = torch.full((R, D), SENT)
    dst = dst0.cuda()
    ops.scatter_rows(src.cuda(), idx.cuda(), dst, src_idx=src_idx.cuda() if gather else None)
    want = dst0.clone()
    want[idx.long()] = src[src_idx.long() if gather else torch.arange(6)].float()
    assert torch.equal(dst.cpu(), want)
    assert torch.equal(fake_ops.scatter_rows(src, idx, dst0.clone(), src_idx=src_idx), want)


def test_store_hidden():
    """hidden[b, state[0] - state[3] - 1] = x[b]; rows before the prompt's end (< 0) and past the buffer (>= max_rows) write nothing"""
    from seedx_b200 import ops
    B, R, D = 5, 12, 5120
    x = torch.randn((B, D), generator=gen(5))
    state = torch.zeros((B, 4), dtype=torch.int32)
    state[:, 3] = torch.tensor([100, 100, 100, 100, 100])
    state[:, 0] = torch.tensor([101, 112, 100, 113, 150])             # rows 0, 11, -1, 12, 49
    h0 = torch.full((B, R, D), SENT)
    h = h0.cuda()
    ops.store_hidden(x.cuda(), state.cuda(), h)
    want = h0.clone()
    want[0, 0], want[1, 11] = x[0], x[1]
    assert torch.equal(h.cpu(), want)
    fh = h0.clone()
    fake_ops.store_hidden(x, state, fh)
    assert torch.equal(fh, want)
