"""Synthetic Llama-shaped decoder stack over the operator surface.

Host-side mirror of the reference's per-layer call sequence -- ExLlamaAttention.fused (model.py:322-417),
ExLlamaMLP.fused (model.py:238-263) for decode, and the unfused path (model.py:419-506, 265-273, 524-552) for
prefill -- expressed only in the reference-facing plugin API (cuda_ext.ext_* / exllama_ext.*) plus the same torch
ops model.py uses for attention.  It exists so that the hot path can be driven and timed end to end on synthetic
GPTQ tensors (no checkpoint, tokenizer or model.py travel to the GPU box); it is not a model implementation:
there is no loader, no sampling, no tokenizer.

Tensor parallelism (new functionality, SURVEY.md 8e): q/k/v and gate/up are column-sharded by whole heads /
group-aligned column blocks, o_proj and down_proj are row-sharded on group boundaries, and the [M, hidden] partial
of each row-parallel projection is summed with ONE all-reduce (exllama_b200/tp.py).
"""
from __future__ import annotations

import math
import torch

from . import capi, cuda_ext
from . import tp as tpmod

ext = cuda_ext.exllama_ext


from .shapes import SHAPES, GQA_SHAPES, LlamaShape  # noqa: E402,F401  (re-exported)


def repeat_kv(x, n_rep):
    """[bsz, kv_heads, seq, head_dim] -> [bsz, kv_heads * n_rep, seq, head_dim], each KV head repeated for the n_rep query heads
    of its group (model.py:310-319)."""
    if n_rep == 1:
        return x
    b, kvh, n, d = x.shape
    return x[:, :, None, :, :].expand(b, kvh, n_rep, n, d).reshape(b, kvh * n_rep, n, d)


class _Arena:
    """One device allocation handed out in 256-byte aligned slices, in request order (a loader that maps one checkpoint file
    region): the GPTQ tensors of a stack then sit back to back in HBM instead of wherever the caching allocator had room."""

    def __init__(self, nbytes, device):
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.off = 0

    def take(self, shape, dtype):
        n = 1
        for d in shape:
            n *= d
        nb = n * torch.empty((), dtype=dtype).element_size()
        v = self.buf[self.off:self.off + nb].view(dtype).view(*shape)
        self.off += (nb + 255) & ~255
        return v

    @staticmethod
    def q4_bytes(K, N, groupsize):
        G = 1 if groupsize is None else K // groupsize
        r = lambda b: (b + 255) & ~255
        return r(K // 8 * N * 4) + r(G * (N // 8) * 4) + r(G * N * 2)


def synth_q4_device(K, N, groupsize, device, gen, act_order=False, scale_lo=None, scale_hi=None, arena=None):
    """Random GPTQ tensor set on the device, shaped like a real checkpoint: uniform 4-bit weights, zero points in the middle of
    the range (stored nibble 6 or 7, i.e. z + 1 = 7 or 8, mean 7.5 = the mean nibble: zero-mean weights, as GPTQ produces for
    symmetric weight groups.  A mean offset of even one quantisation step gives every matrix a DC gain of ~scale * K >> 1 and a
    deep synthetic stack then blows up through its DC mode -- measured: 33B overflowed fp16 within a few layers), and scales sized
    for a per-layer gain below one whatever K is (std(q - z) ~ 4.6, so gain = 4.6 * mean(scale) * sqrt(K) ~ 0.4)."""
    G = 1 if groupsize is None else K // groupsize
    if scale_hi is None:
        scale_hi = 2.3e-3 * (4096.0 / K) ** 0.5
    if scale_lo is None:
        scale_lo = 0.1 * scale_hi
    if arena is not None:
        qweight = arena.take((K // 8, N), torch.int32)
        torch.randint(-2**31, 2**31 - 1, (K // 8, N), dtype=torch.int32, device=device, generator=gen, out=qweight)
    else:
        qweight = torch.randint(-2**31, 2**31 - 1, (K // 8, N), dtype=torch.int32, device=device, generator=gen)
    zn = torch.randint(6, 8, (G, N // 8, 8), dtype=torch.int64, device=device, generator=gen)
    shifts = (torch.arange(8, device=device, dtype=torch.int64) * 4)
    qz = (zn << shifts).sum(-1)                                   # 8 nibbles per word, nibble n % 8 of word [g, n / 8]
    qzeros = torch.where(qz >= 2**31, qz - 2**32, qz).to(torch.int32)
    scales = (torch.rand((G, N), device=device, generator=gen) * (scale_hi - scale_lo) + scale_lo).half()
    if arena is not None:
        qzeros = arena.take((G, N // 8), torch.int32).copy_(qzeros)
        scales = arena.take((G, N), torch.float16).copy_(scales)
    g_idx = None
    if act_order:
        perm = torch.randperm(K, device=device, generator=gen)
        g_idx = torch.empty(K, dtype=torch.int32, device=device)
        g_idx[perm] = 0 if groupsize is None else (torch.arange(K, device=device) // groupsize).int()
        g_idx = g_idx.cpu()
    return qweight, qzeros, scales, g_idx


class Q4Linear:
    """Counterpart of Ex4bitLinear (model.py:130-177): owns the tensors, holds the ext handle."""

    def __init__(self, qweight, qzeros, scales, g_idx, device_index):
        self.qweight, self.qzeros, self.scales, self.g_idx = qweight, qzeros, scales, g_idx
        self.height, self.width = qweight.shape[0] * 8, qweight.shape[1]
        self.q4 = cuda_ext.ext_make_q4(qweight, qzeros, scales, g_idx, device_index)

    def nbytes(self):
        return self.qweight.numel() * 4 + self.qzeros.numel() * 4 + self.scales.numel() * 2

    def forward(self, x, lora=None):
        """x @ W (+ (x @ A) @ B with lora = (A, B), as Ex4bitLinear.forward passes an adapter, model.py:207-217)."""
        if lora is None:
            return cuda_ext.ext_q4_matmul(x, self.q4, self.width)
        return cuda_ext.ext_q4_matmul(x, self.q4, self.width, lora[0], lora[1])


class Layer:
    pass


class DecodeStack:
    def __init__(self, shape: LlamaShape, groupsize=128, act_order=False, device="cuda:0", max_seq=2048,
                 layers=None, seed=0, tp_rank=0, tp_size=1, tp_group=None, with_head=True, batch=1):
        self.shape, self.groupsize, self.act_order = shape, groupsize, act_order
        self.batch = batch                     # sequences the KV caches hold (and the fused plan may step at once)
        self.dplan = None                      # the plan of the last make_plan(), closed by close()
        self.device = torch.device(device)
        self.dev_index = self.device.index or 0
        self.max_seq = max_seq
        self.n_layers = layers if layers is not None else shape.layers
        self.tp_rank, self.tp_size, self.tp_group = tp_rank, tp_size, tp_group
        self.fused_decode_attn = True          # csrc/decode_attn.cu instead of the torch ops of model.py:395-409
        # act-order + tensor parallel (tp.py "act-order checkpoints"): row-parallel shards are cut on group ranges; down's
        # input is local (gate/up column-gathered to match), o_proj's input is the all-gathered attention output indexed
        # by the shard's rows.  The synthetic stack draws every rank's shard directly (a valid local act-order matrix) and
        # a random row set for o_proj, so the work and the exchange are those of a real sharded checkpoint.
        self.o_rows = None
        if shape.kv_heads != shape.heads and tp_size > 1:
            raise NotImplementedError("grouped-query attention under tensor parallelism (KV-head sharding) is not implemented")
        if groupsize is None and tp_size > 1:
            raise NotImplementedError("one quantisation group per matrix (groupsize None) under tensor parallelism is not implemented")
        # groupsize None: one group per matrix, so a single rank's plan takes the whole intermediate width as one unit
        plan = tpmod.plan_shards(shape.hidden, shape.inter, shape.heads, shape.head_dim, groupsize or shape.inter, tp_size)
        self.plan = plan
        h = shape.hidden
        self.local_heads = plan.heads[tp_rank]
        hq = self.local_heads * shape.head_dim
        self.local_kv_heads = shape.kv_heads if tp_size == 1 else self.local_heads
        self.n_rep = self.local_heads // self.local_kv_heads
        hkv = self.local_kv_heads * shape.head_dim
        il = plan.inter_cols[tp_rank][1] - plan.inter_cols[tp_rank][0]
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed * 1000 + tp_rank)                 # this rank's shards
        rep = torch.Generator(device=self.device)
        rep.manual_seed(seed * 1000 + 977)                     # replicated tensors (norms, head): identical on every rank
        with torch.cuda.device(self.device):
            ext.set_tuning_params(8, 2, 8, False, False, False, False, False, False)
            self.layers = []
            per_layer = (_Arena.q4_bytes(h, hq, groupsize) + 2 * _Arena.q4_bytes(h, hkv, groupsize) + _Arena.q4_bytes(hq, h, groupsize) +
                         2 * _Arena.q4_bytes(h, il, groupsize) +
                         _Arena.q4_bytes(il, h, groupsize))
            self.arena = _Arena(per_layer * self.n_layers, self.device)
            for _ in range(self.n_layers):
                L = Layer()
                mk = lambda K, N: Q4Linear(*synth_q4_device(K, N, groupsize, self.device, gen, act_order, arena=self.arena), self.dev_index)
                L.q, L.k, L.v = mk(h, hq), mk(h, hkv), mk(h, hkv)
                L.o = mk(hq, h)
                L.gate, L.up = mk(h, il), mk(h, il)
                L.down = mk(il, h)
                L.ln1 = (1 + 0.05 * torch.randn(h, device=self.device, generator=rep)).half()
                L.ln2 = (1 + 0.05 * torch.randn(h, device=self.device, generator=rep)).half()
                self.layers.append(L)
            if act_order and tp_size > 1:
                g0 = torch.Generator(device="cpu"); g0.manual_seed(seed * 7919 + 13)            # same on every rank
                perm = torch.randperm(h, generator=g0)
                self.o_rows = perm[tp_rank * hq:(tp_rank + 1) * hq].sort().values.to(self.device)
            self.norm = (1 + 0.05 * torch.randn(h, device=self.device, generator=rep)).half()
            self.lm_head = (torch.randn((shape.vocab, h), device=self.device, generator=rep) * 0.02).half() if with_head else None
            # sin/cos tables as model.py:864-877
            inv_freq = 1.0 / (10000.0 ** (torch.arange(0, shape.head_dim, 2, device=self.device).float() / shape.head_dim))
            t = torch.arange(max_seq, device=self.device, dtype=torch.float32)
            freqs = torch.einsum("i,j->ij", t, inv_freq)
            emb = torch.cat((freqs, freqs), dim=-1)
            self.sin = emb.sin()[None, None, :, :].half().contiguous()
            self.cos = emb.cos()[None, None, :, :].half().contiguous()
            # KV cache [batch, kv_heads_local, max_seq, head_dim] per layer (model.py:557-585)
            self.key_cache = [torch.zeros((batch, self.local_kv_heads, max_seq, shape.head_dim), dtype=torch.float16, device=self.device)
                              for _ in range(self.n_layers)]
            self.value_cache = [torch.zeros_like(self.key_cache[0]) for _ in range(self.n_layers)]
            # scratch, as model.py:897-917
            self.temp_state = torch.zeros((max_seq, shape.inter), dtype=torch.float16, device=self.device)
            self.temp_mlp = torch.zeros((4, shape.inter), dtype=torch.float16, device=self.device)
            self.temp_zeros_float = torch.zeros((1, 65536), dtype=torch.float32, device=self.device)
            max_dq = max(max(l.gate.qweight.numel(), l.q.qweight.numel(), l.down.qweight.numel()) for l in self.layers) * 8
            self.temp_dq = torch.zeros((1, max_dq), dtype=torch.float16, device=self.device)
            ext.prepare_buffers(self.device, self.temp_state, self.temp_mlp, self.temp_zeros_float, self.temp_dq)
        self.none = cuda_ext.none_tensor
        self.lora = None                       # per layer None or {projection name: (A [in, r], B [r, out] scaled)}, see add_lora

    # ---- LoRA adapter (lora.py's layout: A transposed to [in, r], B [r, out] pre-scaled by alpha / r) ----------------------------
    PROJ = ("q", "k", "v", "o", "gate", "up", "down")

    def add_lora(self, rank, targets=("q", "v"), layers=None, alpha=None, seed=0):
        """Synthesise one adapter of rank `rank` on the projections `targets` (names of PROJ, or "all") of `layers` (default every
        layer) and attach it to every path of the stack (decode_step, prefill, make_plan).  Zero-mean Gaussian A ~ N(0, 1 / in) and
        B ~ N(0, (0.2 / sqrt(r))^2), then B *= alpha / r as lora.py does (alpha defaults to r): the LoRA term is then about half the
        rms of the projection's own output (synth_q4_device's gain is ~0.4) whatever the rank, and it has no DC gain a deep stack
        could blow up through.  alpha scales the term as it does in PEFT: alpha = 2 r doubles it."""
        if targets == "all":
            targets = self.PROJ
        assert all(t in self.PROJ for t in targets), targets
        alpha = float(rank if alpha is None else alpha)
        g = torch.Generator(device=self.device)
        g.manual_seed(seed * 7717 + 5)
        lora = self.lora or [None] * self.n_layers
        for i in (range(self.n_layers) if layers is None else layers):
            L = self.layers[i]
            ad = dict(lora[i] or {})
            for t in targets:
                lin = getattr(L, t)
                A = (torch.randn((lin.height, rank), device=self.device, generator=g) / math.sqrt(lin.height)).half()
                B = (torch.randn((rank, lin.width), device=self.device, generator=g) * (0.2 / math.sqrt(rank)) * (alpha / rank)).half()
                ad[t] = (A.contiguous(), B.contiguous())
            lora[i] = ad
        self.lora = lora
        return lora

    def _lora_of(self, i, name):
        """(A, B) of projection `name` of layer i, or (none, none)."""
        ad = self.lora[i] if self.lora is not None else None
        if not ad or name not in ad:
            return self.none, self.none
        return ad[name]

    def _lora_temp(self, i, names, rows):
        """lora_temp as model.py:246-252 / 335-341 size it: [1, rows * the largest rank of the call], or none_tensor."""
        r = max([self._lora_of(i, n)[0].shape[1] for n in names if self._lora_of(i, n)[0] is not self.none] + [0])
        return torch.empty((1, rows * r), dtype=torch.float16, device=self.device) if r else self.none

    # ---- bookkeeping for rooflines -------------------------------------------------------------------------
    def q4_weight_bytes_per_token(self):
        """Bytes of every q4 tensor the stack holds (q, k, v, o, gate, up, down of each layer; k and v kv_heads wide)."""
        return sum(l.q.nbytes() + l.k.nbytes() + l.v.nbytes() + l.o.nbytes() + l.gate.nbytes() + l.up.nbytes() + l.down.nbytes()
                   for l in self.layers)

    # ---- decode: fused path, rows == 1 (model.py:528-547) ----------------------------------------------------
    def decode_step(self, hidden, past_len, seq=0):
        """hidden: [1, 1, hidden] fp16 on the device, updated in place layer by layer; returns logits [1, vocab].
        seq: the cache sequence this token belongs to (its rows [0, past_len) are attended, its row past_len is written)."""
        s, none = self.shape, self.none
        bsz, q_len = 1, hidden.shape[1]
        hq = self.local_heads * s.head_dim
        hkv = self.local_kv_heads * s.head_dim
        key_cache = [kc[seq:seq + 1] for kc in self.key_cache]
        value_cache = [vc[seq:seq + 1] for vc in self.value_cache]
        for i, L in enumerate(self.layers):
            q = torch.empty((bsz, q_len, hq), dtype=torch.float16, device=self.device)
            k = torch.empty((bsz, q_len, hkv), dtype=torch.float16, device=self.device)
            v = torch.empty_like(k)
            # LoRA tensors (or none) and lora_temp as ExLlamaAttention.fused passes them (model.py:322-341)
            (q_a, q_b), (k_a, k_b), (v_a, v_b), (o_a, o_b) = (self._lora_of(i, n) for n in ("q", "k", "v", "o"))
            lt_attn = self._lora_temp(i, ("q", "k", "v", "o"), bsz * q_len)
            ext.q4_attn(hidden, L.ln1, s.eps, q, k, v, L.q.q4, L.k.q4, L.v.q4, self.sin, self.cos, q_len, past_len,
                        self.local_heads, self.local_kv_heads, s.head_dim, key_cache[i], value_cache[i], self.max_seq,
                        q_a, q_b, k_a, k_b, v_a, v_b, lt_attn)
            if self.fused_decode_attn and q_len == 1 and s.head_dim == 128:
                # one kernel over the KV cache instead of the five torch launches below (csrc/decode_attn.cu)
                attn = torch.empty_like(q)
                ext.decode_attn(q, key_cache[i], value_cache[i], attn, self.local_heads, self.local_kv_heads,
                                s.head_dim, past_len + 1, self.max_seq)
            else:
                q = q.view(bsz, q_len, self.local_heads, s.head_dim).transpose(1, 2)
                keys = repeat_kv(key_cache[i].narrow(2, 0, past_len + q_len), self.n_rep)
                values = repeat_kv(value_cache[i].narrow(2, 0, past_len + q_len), self.n_rep)
                attn = torch.matmul(q, keys.transpose(2, 3))
                attn /= math.sqrt(s.head_dim)
                attn = torch.nn.functional.softmax(attn, dim=-1, dtype=torch.float16)
                attn = torch.matmul(attn, values).transpose(1, 2).reshape(bsz, q_len, hq)
            x2 = hidden.view(-1, s.hidden)
            if self.tp_size == 1:
                ext.q4_attn_2(x2, attn.view(-1, hq), L.o.q4, o_a, o_b, lt_attn)
                (g_a, g_b), (u_a, u_b), (d_a, d_b) = (self._lora_of(i, n) for n in ("gate", "up", "down"))
                ext.q4_mlp(x2, L.ln2, s.eps, L.gate.q4, L.up.q4, L.down.q4, g_a, g_b, u_a, u_b, d_a, d_b,
                           self._lora_temp(i, ("gate", "up", "down"), bsz * q_len))
            else:
                assert self.lora is None, "LoRA under tensor parallelism is not implemented"
                tpmod.row_parallel_residual(ext, x2, self._o_input(attn.view(-1, hq)), L.o.q4, self.tp_rank, self.tp_group)
                tpmod.mlp_tp(ext, cuda_ext, x2, L, s.eps, self.tp_rank, self.tp_group)
        if self.lm_head is None:
            return hidden
        hn = cuda_ext.ext_rms_norm(hidden, self.norm, s.eps)
        return torch.matmul(hn.view(-1, s.hidden), self.lm_head.t()).float()

    # ---- decode: the whole token as ONE persistent kernel (csrc/decode_step.cu; SURVEY.md 8f-4 / 8f-2) -------------------
    def make_plan(self, with_head=True, max_tokens=None):
        """Build the exl_decode_plan over this stack's handles, norms, caches and tables (borrowed).  max_tokens (1..4): a
        multi-token plan instead, for decode_step_fused_multi (up to max_tokens consecutive tokens of one cache sequence per launch).
        A plan the stack held before stays open: close it, or replace it with slots.open_plan."""
        hs =[[L.q.q4, L.k.q4, L.v.q4, L.o.q4, L.gate.q4, L.up.q4, L.down.q4] for L in self.layers]
        head = self.lm_head if with_head else None
        multi = max_tokens is not None
        if multi and self.lora is not None:
            raise NotImplementedError("LoRA adapters in the multi-token step are not implemented: use prefill")
        self.dplan = capi.DecodePlan(hs, [L.ln1 for L in self.layers], [L.ln2 for L in self.layers], self.key_cache, self.value_cache,
                                    self.sin, self.cos, self.local_heads, self.shape.head_dim, self.max_seq, self.shape.eps,
                                    final_norm=self.norm if head is not None else None, lm_head=head,
                                    tp_rank=self.tp_rank, tp_world=self.tp_size, num_kv_heads=self.local_kv_heads,
                                    max_batch=1 if multi else self.batch, lora=None if multi else self._plan_lora(), max_tokens=max_tokens)
        if multi:
            self._plan_xout = torch.empty((max_tokens, self.shape.hidden), dtype=torch.float16, device=self.device)
            self._plan_logits = torch.empty((max_tokens, self.shape.vocab), dtype=torch.float32, device=self.device) if head is not None else None
            return self.dplan
        if self.tp_size > 1:
            # exchange the cudaIpc handles of the regions the peers reduce into (acc_o, acc_d, cross-barrier counter)
            import torch.distributed as dist
            handles = [None] * self.tp_size
            dist.all_gather_object(handles, self.dplan.ipc_export(), group=self.tp_group)
            self.dplan.ipc_import(handles)
            dist.barrier(self.tp_group)
        self._plan_xout = torch.empty((self.batch, self.shape.hidden) if self.batch > 1 else self.shape.hidden, dtype=torch.float16, device=self.device)
        self._plan_logits = torch.empty((self.batch, self.shape.vocab), dtype=torch.float32, device=self.device) if head is not None else None
        return self.dplan

    def _plan_lora(self):
        """The adapter as DecodePlan takes it: per layer None or a 7-tuple of (A, B) or None; None without an adapter."""
        if self.lora is None:
            return None
        return [None if not ad else tuple(ad.get(n) for n in self.PROJ) for ad in self.lora]

    def decode_step_fused(self, hidden, past_len):
        """hidden: [1, 1, hidden] fp16 (read only).  Returns logits [1, vocab] fp32 (or the final hidden state without a head);
        the final pre-norm hidden state is left in self._plan_xout."""
        self.dplan.step(hidden, past_len, x_out=self._plan_xout, logits=self._plan_logits)
        return self._plan_logits if self._plan_logits is not None else self._plan_xout

    def decode_step_fused_batch(self, hidden, past_lens):
        """One token for each of bsz = len(past_lens) <= batch sequences in one launch: hidden [bsz, 1, hidden] fp16 (read only),
        sequence b at context past_lens[b] of cache sequence b.  Returns logits [bsz, vocab] fp32 (or the final hidden states
        without a head); the final pre-norm hidden states are left in self._plan_xout[:bsz]."""
        bsz = len(past_lens)
        assert hidden.shape[0] == bsz and hidden.is_contiguous(), (hidden.shape, bsz)
        xo = self._plan_xout.view(-1, self.shape.hidden)
        lg = self._plan_logits
        self.dplan.step_batch(hidden, past_lens, x_out=xo, logits=lg)
        return lg[:bsz] if lg is not None else xo[:bsz]

    def decode_step_fused_multi(self, hidden, past_len, seq=0):
        """n <= max_tokens consecutive tokens of cache sequence seq in one launch (a plan from make_plan(max_tokens=...)): hidden
        [n, 1, hidden] fp16 (read only), token t at position past_len + t attending rows [0, past_len) and tokens 0..t of the
        launch -- what prefill(hidden.view(1, n, -1), past_len, seq=seq, last_only=False) computes.  Returns logits [n, vocab] fp32
        (or the final hidden states without a head); the final pre-norm hidden states are left in self._plan_xout[:n]."""
        n = hidden.shape[0]
        assert hidden.numel() == n * self.shape.hidden and hidden.is_contiguous(), hidden.shape
        lg = self._plan_logits
        self.dplan.step_multi(hidden, past_len, seq=seq, x_out=self._plan_xout, logits=lg)
        return lg[:n] if lg is not None else self._plan_xout[:n]

    def _o_input(self, attn_local):
        """o_proj input of this rank: its own heads' output, or -- act-order + TP -- the rows of its group range out of the
        all-gathered attention output (the one extra exchange act-order costs, SURVEY.md 8e hazard 1)."""
        if self.o_rows is None:
            return attn_local
        full = tpmod.all_gather_columns(attn_local, [attn_local.shape[1]] * self.tp_size, self.tp_group)
        return full.index_select(1, self.o_rows)

    # ---- prefill: unfused path (model.py:532-550) --------------------------------------------------------------
    def prefill(self, hidden, past_len=0, last_only=True, seq=0, targets=None):
        """hidden: [bsz, q_len, hidden] fp16; sequence b fills rows [past_len, past_len + q_len) of cache sequence seq + b and attends
        rows [0, past_len + t] of it (a prompt chunk, or a follow-up turn appended to a live cache).  Returns logits [bsz, vocab] of
        the last position (last_only) or [bsz * q_len, vocab].  At past_len 0 attention is torch's causal SDPA (model.py's
        prompt path); at past_len > 0 it is csrc/prefill_attn.cu over the cache in place.
        targets: int64 token ids [bsz, q_len] (or any shape of bsz * q_len).  Then the head is rms_norm + exl_token_logprobs over every
        position (last_only does not apply) and the call returns (logprob fp32 [bsz * q_len], greedy int64 [bsz * q_len]) instead of
        logits (scoring.token_logprobs)."""
        s = self.shape
        bsz, q_len, _ = hidden.shape
        if targets is not None:
            self._check_targets(targets, bsz * q_len)
        if bsz > self.batch:
            raise ValueError(f"prefill of {bsz} sequences into caches that hold {self.batch} (DecodeStack(..., batch=))")
        if seq < 0 or seq + bsz > self.batch:
            raise ValueError(f"prefill of {bsz} sequences into cache sequences [{seq}, {seq + bsz}): the caches hold [0, {self.batch})")
        if past_len < 0 or past_len + q_len > self.max_seq:
            raise ValueError(f"prefill of {q_len} tokens at past_len {past_len}: rows [{past_len}, {past_len + q_len}) do not fit "
                             f"max_seq {self.max_seq}")
        if past_len > 0 and self.tp_size > 1:
            raise NotImplementedError("prefill at past_len > 0 under tensor parallelism is not implemented")
        hq = self.local_heads * s.head_dim
        kvh = self.local_kv_heads
        ad = lambda i, n: (self.lora[i] or {}).get(n) if self.lora is not None else None      # (A, B) or None
        for i, L in enumerate(self.layers):
            key_cache, value_cache = self.key_cache[i][seq:seq + bsz], self.value_cache[i][seq:seq + bsz]
            residual = hidden
            x = cuda_ext.ext_rms_norm(hidden, L.ln1, s.eps)
            q = L.q.forward(x, ad(i, "q"))
            k = L.k.forward(x, ad(i, "k"))
            ext.rope_(q, self.sin, self.cos, past_len, self.local_heads, s.head_dim)
            ext.rope_(k, self.sin, self.cos, past_len, kvh, s.head_dim)
            k = k.view(bsz, q_len, kvh, s.head_dim).transpose(1, 2)
            v = L.v.forward(x, ad(i, "v")).view(bsz, q_len, kvh, s.head_dim).transpose(1, 2)
            key_cache.narrow(2, past_len, q_len).copy_(k)
            value_cache.narrow(2, past_len, q_len).copy_(v)
            if past_len > 0:
                # one kernel over the cache in place instead of repeat_kv + the additive mask + SDPA (csrc/prefill_attn.cu): q stays
                # [bsz, q_len, heads, hd] as rope_ left it, and the output is already o_proj's input layout
                attn = torch.empty((bsz, q_len, hq), dtype=torch.float16, device=self.device)
                ext.prefill_attn(q, key_cache, value_cache, attn, self.local_heads, kvh, s.head_dim, past_len, self.max_seq)
            else:
                q = q.view(bsz, q_len, self.local_heads, s.head_dim).transpose(1, 2)
                keys = repeat_kv(key_cache.narrow(2, 0, past_len + q_len), self.n_rep)
                values = repeat_kv(value_cache.narrow(2, 0, past_len + q_len), self.n_rep)
                attn = torch.nn.functional.scaled_dot_product_attention(q, keys, values, attn_mask=None, is_causal=True)
                attn = attn.transpose(1, 2).reshape(bsz, q_len, hq)
            o = L.o.forward(self._o_input(attn.view(-1, hq)).view(bsz, q_len, hq), ad(i, "o"))
            if self.tp_size > 1:
                tpmod.all_reduce(o, self.tp_group)
            hidden = residual + o
            residual = hidden
            x = cuda_ext.ext_rms_norm(hidden, L.ln2, s.eps)
            y = torch.nn.functional.silu(L.gate.forward(x, ad(i, "gate")))
            y *= L.up.forward(x, ad(i, "up"))
            y = L.down.forward(y, ad(i, "down"))
            if self.tp_size > 1:
                tpmod.all_reduce(y, self.tp_group)
            hidden = residual + y
        if self.lm_head is None:
            return hidden
        if targets is not None:
            return self._token_logprobs(hidden, targets)
        if last_only:
            hidden = hidden[:, -1:, :].contiguous()
        hn = cuda_ext.ext_rms_norm(hidden, self.norm, s.eps)
        return torch.matmul(hn.view(-1, s.hidden), self.lm_head.t()).float()

    def _check_targets(self, targets, n):
        if self.lm_head is None:
            raise ValueError("targets given to a stack without a head (with_head=False)")
        if not isinstance(targets, torch.Tensor) or targets.dtype != torch.int64 or targets.numel() != n or targets.device != self.device:
            raise ValueError(f"targets must be an int64 tensor of {n} token ids on {self.device}, got "
                             f"{getattr(targets, 'dtype', type(targets))} {tuple(getattr(targets, 'shape', ()))}")

    def _token_logprobs(self, hidden, targets):
        """The head of prefill(targets=) / prefill_ragged(targets=): rms_norm of every position, then exl_token_logprobs."""
        from . import scoring
        hn = cuda_ext.ext_rms_norm(hidden, self.norm, self.shape.eps)
        return scoring.token_logprobs(hn.view(-1, self.shape.hidden), self.lm_head, targets.reshape(-1).contiguous())

    def prefill_ragged(self, hidden, q_lens, past_lens, seqs=None, last_only=True, targets=None):
        """n prompts or follow-up turns of different lengths at different past_lens in one call.  hidden: [T, hidden] fp16, the
        sequences' tokens packed in order (sequence i owns rows [sum(q_lens[:i]), + q_lens[i])); sequence i fills rows
        [past_lens[i], past_lens[i] + q_lens[i]) of cache sequence seqs[i] (default 0 .. n-1, distinct) and attends rows
        [0, past_lens[i] + t] of it.  The same results as n prefill(x_i, past_lens[i], seq=seqs[i]) calls except for the GEMM route:
        the q4 GEMMs run once per layer on all T rows.  Per layer one rope_cache_ragged and one prefill_attn_ragged launch
        (csrc/elementwise.cu, csrc/prefill_attn.cu).  Returns the logits [n, vocab] of each sequence's last token (last_only) or
        [T, vocab].  targets: int64 token ids [T], packed as hidden is; then the call returns (logprob fp32 [T], greedy int64 [T]) of
        every position instead of logits, as prefill(targets=) does."""
        s = self.shape
        if self.tp_size > 1:
            raise NotImplementedError("prefill_ragged under tensor parallelism is not implemented")
        q_lens, past_lens = [int(v) for v in q_lens], [int(v) for v in past_lens]
        n = len(q_lens)
        seqs = list(range(n)) if seqs is None else [int(v) for v in seqs]
        if not 1 <= n <= capi.RAGGED_MAX_SEQ:
            raise ValueError(f"prefill_ragged of {n} sequences: one call takes 1 .. {capi.RAGGED_MAX_SEQ}")
        if len(past_lens) != n or len(seqs) != n:
            raise ValueError(f"prefill_ragged: {n} q_lens, {len(past_lens)} past_lens and {len(seqs)} seqs")
        for ql, pl, sq in zip(q_lens, past_lens, seqs):
            if ql < 1:
                raise ValueError(f"prefill of {ql} tokens: q_len must be at least 1")
            if pl < 0 or pl + ql > self.max_seq:
                raise ValueError(f"prefill of {ql} tokens at past_len {pl}: rows [{pl}, {pl + ql}) do not fit max_seq {self.max_seq}")
            if not 0 <= sq < self.batch:
                raise ValueError(f"prefill into cache sequence {sq}: the caches hold [0, {self.batch}) (DecodeStack(..., batch=))")
        if len(set(seqs)) != n:
            raise ValueError(f"prefill_ragged into cache sequences {seqs}: a cache sequence is named twice")
        T = sum(q_lens)
        if hidden.dim() != 2 or tuple(hidden.shape) != (T, s.hidden):
            raise ValueError(f"prefill_ragged: hidden {tuple(hidden.shape)} is not [sum(q_lens) = {T}, {s.hidden}]")
        if targets is not None:
            self._check_targets(targets, T)
        hq = self.local_heads * s.head_dim
        kvh = self.local_kv_heads
        ad = lambda i, n: (self.lora[i] or {}).get(n) if self.lora is not None else None      # (A, B) or None
        hidden = hidden.view(1, T, s.hidden)
        for i, L in enumerate(self.layers):
            residual = hidden
            x = cuda_ext.ext_rms_norm(hidden, L.ln1, s.eps)
            q = L.q.forward(x, ad(i, "q"))
            k = L.k.forward(x, ad(i, "k"))
            v = L.v.forward(x, ad(i, "v"))
            ext.rope_cache_ragged(q, k, v, self.key_cache[i], self.value_cache[i], self.sin, self.cos, q_lens, past_lens, seqs,
                                  self.local_heads, kvh, s.head_dim, self.max_seq)
            attn = torch.empty((1, T, hq), dtype=torch.float16, device=self.device)
            ext.prefill_attn_ragged(q, self.key_cache[i], self.value_cache[i], attn, q_lens, past_lens, seqs, self.local_heads, kvh,
                                    s.head_dim, self.max_seq)
            hidden = residual + L.o.forward(attn, ad(i, "o"))
            residual = hidden
            x = cuda_ext.ext_rms_norm(hidden, L.ln2, s.eps)
            y = torch.nn.functional.silu(L.gate.forward(x, ad(i, "gate")))
            y *= L.up.forward(x, ad(i, "up"))
            hidden = residual + L.down.forward(y, ad(i, "down"))
        if self.lm_head is None:
            return hidden.view(T, s.hidden)
        if targets is not None:
            return self._token_logprobs(hidden, targets)
        if last_only:
            ends, t = [], 0
            for ql in q_lens:
                t += ql
                ends.append(t - 1)
            hidden = hidden[:, torch.tensor(ends, device=self.device), :].contiguous()
        hn = cuda_ext.ext_rms_norm(hidden, self.norm, s.eps)
        return torch.matmul(hn.view(-1, s.hidden), self.lm_head.t()).float()

    def close(self):
        if self.dplan is not None:
            self.dplan.close()
        ext.cleanup()
