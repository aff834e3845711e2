"""Continuous batching of the LLaMA token loop (`ContinuousBatcher`) and of the de-tokenizer's denoising loop (`DenoiseBatcher`, below).

`ContinuousBatcher`: continuous batching of the LLaMA token loop (SURVEY.md §8 f-3): requests are admitted into free sequence slots BETWEEN replays of the
lock-step decode graph instead of only at the start of a batch.

The reference decodes one request at a time with HF `generate` (src/models/mllm/seed_x.py:184-189); `LlamaForCausalLM.generate_greedy_batch`
already streams the weights once per step for up to 8 requests that start together.  What makes admission in the middle cheap here is that every
piece of per-request state the captured graph reads is a row of a static device buffer (`seq`, `state`, the page table, the harvest buffer): a
new request is a prefill into one slot's pages plus a few row writes, the graph is neither re-captured nor aware of it.  A retired or idle slot is
parked by a non-zero `state[slot][1]` (seedx_logits_argmax): it keeps riding along in the batched GEMVs — the weights are read anyway — but its
sequence, KV length and harvest row no longer move.

Results are those of running every request alone in the same engine: slots never read each other's rows
(`tests/test_llm_host_cpu.py::test_continuous_batching_equals_isolated_runs`, `tests/test_llm_gpu.py::test_continuous_batching_gpu`)."""
import collections

import torch

from . import _lib, ops
from ._lib import SeedxError
from .llm import GreedyOutput
from .sampler import _copy_tree, _same_layout, decode_to_uint8


class ContinuousBatcher:
    PARKED = -1          # state[slot][1] of a slot without a live request

    def __init__(self, llm, slots=4, img_ids=None, eos_id=None, use_graph=True):
        if slots not in (1, 2, 4, 8):
            raise SeedxError("slots must be 1, 2, 4 or 8 (the batched GEMV variants)")
        self.llm, self.n_slots, self.eos_id, self.use_graph = llm, slots, eos_id, use_graph
        dev = llm.device
        llm._alloc_state(slots)
        self.img_key = tuple(int(i) for i in img_ids) if img_ids is not None else None
        self.img_dev = torch.tensor(list(self.img_key), dtype=torch.int32, device=dev) if self.img_key is not None else None
        llm._img_key, llm._img_dev = self.img_key, self.img_dev
        llm._hidden = torch.zeros((slots, llm.max_len, llm.cfg["hidden"]), device=dev, dtype=torch.float32)
        self.hidden = llm._hidden
        self.pending = collections.deque()
        self.live = [None] * slots            # per slot: dict(rid, P, ahead, budget)
        self.graph = None
        self.next_rid = 0
        self.steps = 0
        st = torch.zeros((slots, 4), dtype=torch.int32)
        st[:, 0], st[:, 1], st[:, 3] = 1, self.PARKED, 1          # parked: length 1 (a valid cache row), nothing appended
        llm.state.copy_(st)
        for s in range(slots):
            llm.reserve_kv(s, 1, fresh=True)

    # ---- requests --------------------------------------------------------------------------------------------------------------
    def submit(self, input_ids, inputs_embeds, max_new_tokens):
        """queue a request (prompt ids [P], prompt embeddings [P, D]); returns its id"""
        ids = torch.as_tensor(input_ids).reshape(-1)
        if ids.numel() + max_new_tokens > self.llm.max_len:
            raise SeedxError("prompt + max_new_tokens exceeds the KV cache")
        rid = self.next_rid
        self.next_rid += 1
        self.pending.append(dict(rid=rid, ids=ids, emb=inputs_embeds.reshape(ids.numel(), -1), budget=int(max_new_tokens)))
        return rid

    def _admit(self, slot, req):
        """prefill one slot and write its rows of the static state: exactly what generate_greedy_batch does for every slot at the start of a batch,
        including the jump-forward over a forced image span"""
        llm, dev = self.llm, self.llm.device
        ids, emb = req["ids"], req["emb"].to(dev, torch.float32)
        P = ids.numel()
        ahead = []
        last = int(ids[-1])
        if llm.jump_forward and self.img_key is not None and last in self.img_key[:-1]:
            ahead = list(self.img_key[self.img_key.index(last) + 1:])[: max(req["budget"] - 1, 0)]
        llm.seq[slot, :P].copy_(ids.to(dev, torch.int32))
        if ahead:
            a_t = torch.tensor(ahead, dtype=torch.int32, device=dev)
            llm.seq[slot, P:P + len(ahead)].copy_(a_t)
            emb = torch.cat([emb, llm.get_input_embeddings()(a_t)[0]], dim=0)
        xs = llm.prefill(emb, slot=slot)                              # fresh=True inside: the slot's old pages go back to the pool first
        llm.reserve_kv(slot, P + req["budget"])
        na = len(ahead)
        ops.gemv(llm.lm_head, xs[P + na - 1], llm.logits[slot], rms_w=llm.norm, eps=llm.cfg["eps"])
        if na:
            ops.layernorm(xs[P:P + na], llm.norm, None, llm.cfg["eps"], out=self.hidden[slot, :na], rms=True)
        llm.state[slot].copy_(torch.tensor([P + na, 0, na, P], dtype=torch.int32))
        # first generated token of this slot only (the other slots' rows must not move): the batched kernel on a one-row view
        ops.logits_argmax(llm.logits[slot:slot + 1], self.img_dev, llm.seq[slot:slot + 1], llm.state[slot:slot + 1], self.eos_id, False)
        self.live[slot] = dict(rid=req["rid"], P=P, budget=req["budget"])

    def _retire(self, slot, n_gen):
        llm, r = self.llm, self.live[slot]
        P = r["P"]
        seq = llm.seq[slot, :P + n_gen].to(torch.int64).cpu().unsqueeze(0)
        out = GreedyOutput(seq, self.hidden[slot, :max(n_gen - 1, 0)].clone(), n_gen)
        out.prefill_hidden = None
        llm.state[slot].copy_(torch.tensor([1, self.PARKED, 0, 1], dtype=torch.int32))       # park: the next admission overwrites everything
        self.live[slot] = None
        return r["rid"], out

    # ---- the loop --------------------------------------------------------------------------------------------------------------
    def _replay(self):
        llm = self.llm
        if not self.use_graph:
            llm._decode_step(self.hidden, self.img_dev, self.eos_id, False)
            return
        if self.graph is None:
            s_ = torch.cuda.Stream()
            s_.wait_stream(torch.cuda.current_stream())
            self.graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            # capturing executes nothing: the state the first replay reads is the one the admissions below have written
            with torch.cuda.graph(self.graph, stream=s_):
                llm._decode_step(self.hidden, self.img_dev, self.eos_id, False)
            self.graph.n_kernels = _lib.launch_count() - n0
            torch.cuda.current_stream().wait_stream(s_)
        self.graph.replay()
        _lib.note_replay(self.graph.n_kernels)

    def step(self):
        """admit waiting requests into free slots, retire what is complete, run one token step for all slots.  Returns the finished
        (request id, GreedyOutput) pairs."""
        llm = self.llm
        for s in range(self.n_slots):
            if self.live[s] is None and self.pending:
                self._admit(s, self.pending.popleft())
        done = []
        st = llm.state.cpu().tolist()                   # one small read per step: lengths and EOS marks of all slots
        for s in range(self.n_slots):
            r = self.live[s]
            if r is None:
                continue
            n_gen = st[s][2]
            if st[s][1] > 0:                            # EOS produced: stop at (and include) it, like HF greedy_search
                done.append(self._retire(s, min(st[s][1], r["budget"])))
            elif n_gen >= r["budget"]:
                done.append(self._retire(s, r["budget"]))
        if any(r is not None for r in self.live):
            self._replay()
            self.steps += 1
        return done

    def idle(self):
        return not self.pending and all(r is None for r in self.live)

    def run(self, arrivals=None):
        """drive the loop until everything submitted has finished.  arrivals: optional {step index: [(ids, emb, max_new_tokens), ...]} submitted when
        the loop reaches that step (staggered arrivals for tests / load generators).  Returns {request id: GreedyOutput}."""
        arrivals = dict(arrivals or {})
        results, i = {}, 0
        while arrivals or not self.idle():
            for a in arrivals.pop(i, []):
                self.submit(*a)
            for rid, out in self.step():
                results[rid] = out
            i += 1
            if i > 100000:
                raise SeedxError("ContinuousBatcher.run: no progress")
        return results


class DenoiseBatcher:
    """Continuous batching of the de-tokenizer's denoising loop: image requests are admitted into free UNet slots BETWEEN replays of one captured
    graph (the UNet forward over all slots + seedx_cfg_euler_slots), each with its own step count, guidance, image guidance and seed.

    `sampler.DenoiseLoop` runs a batch lock-step: a request that arrives one step late waits for the whole batch, and requests with different
    `num_inference_steps` or guidance cannot share one.  Here every per-request quantity the graph reads is a row of a static device buffer:
      x [S,4,h,w], unet_in [br*S,h,w,8], t_dev [br*S]       sampler state, UNet input and per-row timestep (row br*S + s)
      state int32 [S,2]                                     (step index, step count); a slot is live while index < count
      sig [S,max_steps+1], ts [S,max_steps], scal [S,3]     its sigma / timestep tables and (guidance, image guidance, init_noise_sigma)
      ctx / text_embeds / time_ids [br*S, ...] and cond     conditioning rows and the prepare_cond output the graph reads
    Every kernel of the UNet forward is batch-row independent (GroupNorm per image, LayerNorm and FP8 activation scales per row / image), so a
    slot gets the bits `DenoiseLoop` at batch S gives the same request in the same slot, whatever the other slots hold.

    Admission (FIFO into the lowest free slot): the slot's table rows from scheduler.set_timesteps(n), its conditioning rows and edit latents,
    prepare_cond recomputed over all S slots (the hoisted K/V GEMMs keep DenoiseLoop's shapes, hence its bits) and copied into the captured cond,
    then the initialisation of that slot.  The host knows every schedule, so it retires a slot after the replay that made its last update
    without reading anything back; a retired slot is parked (count 0, UNet input rows zeroed so the forward keeps reading finite values) and
    rides along in the forward until the next admission."""

    def __init__(self, adapter, slots=4, height=1024, width=1024, max_steps=100, output_type="uint8", use_graph=True):
        if not 1 <= slots <= 64:
            raise SeedxError("slots must be between 1 and 64")
        if max_steps < 1:
            raise SeedxError("max_steps must be >= 1")
        if output_type not in ("uint8", "latent", "pil"):
            raise SeedxError(f"output_type {output_type!r}: expected 'uint8', 'latent' or 'pil'")
        if height % 8 or width % 8:
            raise SeedxError("height and width must be multiples of 8")
        self.ad, self.unet, self.sch = adapter, adapter.unet, adapter.scheduler
        self.vae = getattr(adapter, "vae", None)
        self.branches = adapter.branches
        if self.branches not in (2, 3):
            raise SeedxError("the adapter must have 2 (t2i) or 3 (edit) branches")
        if self.branches == 3 and self.unet.cfg["in_channels"] != 8:
            raise SeedxError("an edit adapter needs the 8-channel conv_in checkpoint (adapter_modules.py:183-198)")
        self.S, self.max_steps, self.H, self.W = slots, max_steps, height, width
        self.output_type, self.use_graph = output_type, use_graph
        dev = self.unet.device
        S, nb, h, w = slots, self.branches, height // 8, width // 8
        self.latent_hw = (h, w)
        self.x = torch.zeros((S, 4, h, w), device=dev, dtype=torch.float32)
        self.unet_in = torch.zeros((nb * S, h, w, 8), device=dev, dtype=torch.float16)
        self.t_dev = torch.zeros((nb * S,), device=dev, dtype=torch.float32)
        self.state = torch.zeros((S, 2), device=dev, dtype=torch.int32)
        self.sig = torch.zeros((S, max_steps + 1), device=dev, dtype=torch.float32)
        self.ts = torch.zeros((S, max_steps), device=dev, dtype=torch.float32)
        self.scal = torch.zeros((S, 3), device=dev, dtype=torch.float32)
        self.time_ids = torch.tensor([[height, width, 0, 0, height, width]], dtype=torch.float32, device=dev).repeat(nb * S, 1)
        self.ctx = self.text_embeds = None            # allocated at the first admission (token count / widths come from the resampler)
        self.cond = None
        self.graph = None
        self.graph_kernels = 0
        self.captures = 0
        self.eps = None
        self.pending = collections.deque()
        self.live = [None] * S                        # per slot: dict(rid, n, done)
        self.slot_of = {}                             # request id -> the slot it was admitted into
        self.next_rid = 0
        self.steps = 0

    # ---- requests --------------------------------------------------------------------------------------------------------------
    def submit(self, image_embeds, num_inference_steps=50, guidance_scale=7.5, image_guidance_scale=1.5, seed=None, latents=None,
               latent_image=None, input_image_size=448):
        """queue one image request (image_embeds [1, tokens, dim] or [tokens, dim]); the keywords mean what they mean in adapter.generate.
        Returns its id; raises SeedxError (and queues nothing) for a request this batcher cannot serve."""
        n = num_inference_steps
        if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= self.max_steps:
            raise SeedxError(f"num_inference_steps={n!r}: expected an integer in 1..{self.max_steps}")
        if latent_image is not None and self.branches != 3:
            raise SeedxError("latent_image needs the edit adapter (SDXLAdapterWithLatentImage)")
        emb = image_embeds if image_embeds.dim() == 3 else image_embeds.unsqueeze(0)
        if emb.dim() != 3 or emb.shape[0] != 1:
            raise SeedxError("image_embeds must hold one request: [1, tokens, dim] or [tokens, dim]")
        if latents is not None and tuple(latents.shape) != (1, 4) + self.latent_hw:
            raise SeedxError(f"latents of shape {tuple(latents.shape)}: expected {(1, 4) + self.latent_hw}")
        rid = self.next_rid
        self.next_rid += 1
        self.pending.append(dict(rid=rid, emb=emb, n=n, g=float(guidance_scale), ig=float(image_guidance_scale), seed=seed, latents=latents,
                                 latent_image=latent_image, image_size=input_image_size))
        return rid

    def _write_rows(self, slot, req):
        """the slot's rows of every static buffer except cond: conditioning, edit latents, noise, schedule tables and state"""
        ad, S, nb, dev = self.ad, self.S, self.branches, self.unet.device
        p, neg, pp, npool = ad.get_image_embeds(image_embeds=req["emb"], return_negative=True, image_size=req["image_size"])
        rows = ((neg, npool), (p, pp)) if nb == 2 else ((p, pp), (neg, npool), (neg, npool))   # [negative, positive] / [text, image, uncond]
        if self.ctx is None:
            self.ctx = torch.zeros((nb * S,) + tuple(p.shape[1:]), device=dev, dtype=p.dtype)
            self.text_embeds = torch.zeros((nb * S,) + tuple(pp.shape[1:]), device=dev, dtype=pp.dtype)
        if tuple(p.shape[1:]) != tuple(self.ctx.shape[1:]) or tuple(pp.shape[1:]) != tuple(self.text_embeds.shape[1:]):
            raise SeedxError("every request of a DenoiseBatcher must give the same conditioning shape")
        for br, (c, t) in enumerate(rows):
            self.ctx[br * S + slot].copy_(c[0])
            self.text_embeds[br * S + slot].copy_(t[0])
        if nb == 3:
            H, W = self.H, self.W
            il = ad._image_latents(req["latent_image"], H, W) if req["latent_image"] is not None else \
                torch.zeros((1, 4) + self.latent_hw, device=dev)
            il16 = ops.nchw_to_nhwc_f16(il.float().contiguous(), 4)                  # [1,h,w,4] fp16, as DenoiseLoop.set_condition
            for br in range(2):
                ops.unary_f16(il16.view(-1, 4), out=self.unet_in[br * S + slot].view(-1, 8)[:, 4:8])
            self.unet_in[2 * S + slot, ..., 4:].zero_()
        noise = ad._noise(1, self.H, self.W, req["seed"], req["latents"])
        self.x[slot].copy_(noise[0])
        n = req["n"]
        sch = self.sch.set_timesteps(n)              # shared with the adapter and mutated by set_timesteps: copy what this slot needs
        sig = torch.zeros((self.max_steps + 1,), dtype=torch.float32)
        ts = torch.zeros((self.max_steps,), dtype=torch.float32)
        sig[:n + 1] = torch.tensor(list(sch.sigmas), dtype=torch.float32)
        ts[:n] = torch.tensor(list(sch.timesteps), dtype=torch.float32)
        self.sig[slot].copy_(sig)
        self.ts[slot].copy_(ts)
        self.scal[slot].copy_(torch.tensor([req["g"], req["ig"], sch.init_noise_sigma], dtype=torch.float32))
        self.state[slot].copy_(torch.tensor([0, n], dtype=torch.int32))
        self.live[slot] = dict(rid=req["rid"], n=n, done=0)
        self.slot_of[req["rid"]] = slot

    def _refresh_cond(self):
        cond = self.unet.prepare_cond(self.ctx, self.text_embeds, self.time_ids)
        if self.cond is None:
            self.cond = cond
        elif _same_layout(self.cond, cond):
            _copy_tree(self.cond, cond)               # same buffers, new values: the captured graph stays valid
        else:
            raise SeedxError("DenoiseBatcher: the conditioning layout changed under a captured graph")

    def _admit(self):
        fresh = []
        for s in range(self.S):
            if self.live[s] is None and self.pending:
                self._write_rows(s, self.pending.popleft())
                fresh.append(s)
        if fresh:
            self._refresh_cond()
            ops.cfg_euler_slots(None, self.x, self.unet_in, self.t_dev, self.state, self.sig, self.ts, self.scal, self.branches, fresh=fresh)
        return fresh

    def _retire(self, slot):
        r = self.live[slot]
        lat = self.x[slot:slot + 1].clone()
        self.state[slot].zero_()                      # park: count 0, the slot step leaves it alone
        for br in range(self.branches):
            self.unet_in[br * self.S + slot].zero_()
        self.live[slot] = None
        if self.output_type == "latent":
            return r["rid"], lat
        u8 = decode_to_uint8(self.vae, lat)
        return r["rid"], (u8 if self.output_type == "uint8" else self.ad._to_pil(u8)[0])

    # ---- the loop --------------------------------------------------------------------------------------------------------------
    def _step_work(self):
        self.eps = self.unet.forward_nhwc(self.unet_in, self.t_dev, self.cond)
        ops.cfg_euler_slots(self.eps, self.x, self.unet_in, self.t_dev, self.state, self.sig, self.ts, self.scal, self.branches)

    def _replay(self):
        if not self.use_graph:
            self._step_work()
            return
        if self.graph is None:
            s_ = torch.cuda.Stream()
            s_.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s_):
                self.unet.forward_nhwc(self.unet_in, self.t_dev, self.cond)   # warm-up outside capture (lazy one-time setup in the library)
            torch.cuda.current_stream().wait_stream(s_)
            self.graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            # capturing executes nothing: the first replay reads the state the admissions have written
            with torch.cuda.graph(self.graph):
                self._step_work()
            self.graph_kernels = _lib.launch_count() - n0
            self.captures += 1
        self.graph.replay()
        _lib.note_replay(self.graph_kernels)

    def step(self):
        """admit waiting requests into free slots, run one denoising step of every live slot (one graph replay), retire the slots that made
        their last step.  Returns the finished (request id, output) pairs."""
        self._admit()
        done = []
        if any(r is not None for r in self.live):
            self._replay()
            self.steps += 1
            for s, r in enumerate(self.live):
                if r is not None:
                    r["done"] += 1
                    if r["done"] == r["n"]:
                        done.append(self._retire(s))
        return done

    def idle(self):
        return not self.pending and all(r is None for r in self.live)

    def run(self, arrivals=None):
        """drive the loop until everything submitted has finished.  arrivals: optional {step index: [request, ...]} submitted when the loop
        reaches that step; a request is a dict of submit() keywords or a tuple of its positional arguments.  Returns {request id: output}."""
        arrivals = dict(arrivals or {})
        results, i = {}, 0
        while arrivals or not self.idle():
            for a in arrivals.pop(i, []):
                if isinstance(a, dict):
                    self.submit(**a)
                else:
                    self.submit(*a)
            for rid, out in self.step():
                results[rid] = out
            i += 1
            if i > 10000000:
                raise SeedxError("DenoiseBatcher.run: no progress")
        return results
