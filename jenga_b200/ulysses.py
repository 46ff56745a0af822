"""Ulysses sequence parallelism around the carved-attention operator (one box, NVLink/NVSwitch).

Drop-in for the reference's SP wrapper
  hyvideo/modules/xdit_ring_atten.py:61-222  xFuserLongContextAttention.forward
  hyvideo/modules/attenion.py:159-195        my_parallel_attention
Outside attention each rank owns a contiguous 1/P slice of the curve-ordered image tokens and
a replica of the text tokens; inside, rank r owns heads [r*H/P, (r+1)*H/P) over the whole
sequence.  Data movement (SURVEY Appendix A2):
  in : Q, K, V image rows   all-to-all (scatter heads, gather sequence)       — 3 collectives
       text Q/K/V           local head slice (the reference's text-Q all-to-all returns
                            exactly that slice, :129-131 — no exchange needed)
  out: image rows           all-to-all (scatter sequence, gather heads)       — 1 collective
       text rows            all-gather over heads (the reference repeats the rows P times and
                            all-to-alls them, :207,:215-217 — same result)
Collectives are NCCL via torch.distributed (`gloo` works for the CPU tests of the layout
logic); the attention itself is the single-GPU operator on the rank's head group.

Three keyword arguments serve the Hilbert-sharded Wan forward (wan_sp.py); their defaults leave every
other call as it was:
  first_frame_blocks  handed to the operator (the Wan first-frame rule, wan/…:400-406)
  dense               no selection: the dense class of the attention kernel over all rows, exactly
                      as the flash_attn shim runs it on one GPU (the Wan warm-up steps,
                      model_mul.py:153), following attention.QK_INT8 / PV_FP8 the same way
  seq_len             the global valid length L when the ranks' equal slices are zero-padded
                      (P*n_loc > L): the operator sees the first L rows only, so its blocks, pooling
                      and limits are those of one GPU; the result rows past L are zero
"""
from __future__ import annotations

import torch
import torch.distributed as dist

BLOCK = 128


def _group_size_rank(group):
    return dist.get_world_size(group), dist.get_rank(group)


def seq_to_heads(x: torch.Tensor, group=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """[B, n_loc, H, D] (all heads, my token slice) -> [B, P*n_loc, H/P, D] (my heads, all
    tokens, slices concatenated in rank order).  == SeqAllToAll4D(scatter_idx=2, gather_idx=1)."""
    P, _ = _group_size_rank(group)
    B, n, H, D = x.shape
    assert H % P == 0, "heads must divide by the SP degree"
    h = H // P
    send = x.reshape(B, n, P, h, D).permute(2, 0, 1, 3, 4).contiguous()  # [P, B, n, h, D]
    if B == 1 and out is not None and out.is_contiguous():
        # rank-order concatenation along the sequence IS the receive layout: land in place
        dist.all_to_all_single(out.view(P, 1, n, h, D), send, group=group)
        return out
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    y = recv.permute(1, 0, 2, 3, 4).reshape(B, P * n, h, D)  # view when B == 1
    if out is not None:
        out.copy_(y)
        return out
    return y


def heads_to_seq(x: torch.Tensor, group=None) -> torch.Tensor:
    """[B, P*n_loc, H/P, D] -> [B, n_loc, H, D].  == SeqAllToAll4D(scatter_idx=1, gather_idx=2)."""
    P, _ = _group_size_rank(group)
    B, N, h, D = x.shape
    assert N % P == 0
    n = N // P
    send = x.reshape(B, P, n, h, D).permute(1, 0, 2, 3, 4).contiguous()  # [P, B, n, h, D]
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    return recv.permute(1, 2, 0, 3, 4).reshape(B, n, P * h, D)


def _valid_rows(seq_len, N, n, T, dense, first_frame_blocks):
    """L, the rows the operator sees (the seq_len / dense / first_frame_blocks arguments checked)"""
    L = N if seq_len is None else int(seq_len)
    if not N - n < L <= N:
        raise ValueError(f"seq_len {L} does not fit {N // n} slices of {n} rows with a real row in each")
    if (L != N or dense) and T:
        raise ValueError("seq_len < P * n_loc and dense are built for image rows alone (no joint tensors)")
    if dense and first_frame_blocks:
        raise ValueError("a dense call has no selection: first_frame_blocks must be 0")
    return L


def _dense_shim(q, k, v):
    """the single-GPU dense call of the Wan self-attention (the flash_attn_varlen_func shim over one
    segment of all rows)"""
    from .flash_attn_shim import flash_attn_func
    return flash_attn_func(q, k, v)


def gather_heads(x: torch.Tensor, group=None) -> torch.Tensor:
    """[B, T, H/P, D] on every rank (different head groups) -> [B, T, H, D] everywhere."""
    P, _ = _group_size_rank(group)
    B, T, h, D = x.shape
    recv = torch.empty((P * B, T, h, D), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(recv, x.contiguous(), group=group)
    return recv.view(P, B, T, h, D).permute(1, 2, 0, 3, 4).reshape(B, T, P * h, D)


class UlyssesCarvedAttention:
    """Callable with the signature the DiT blocks use for `hybrid_seq_parallel_attn`
    (xdit_ring_atten.py:61-85).  `attn_fn` and `dense_fn` (q, k, v -> out, the dense=True call) are
    injectable so the CPU tests can exercise the layout logic with the oracle; by default they are
    the sm_90a operator and the flash_attn shim."""

    def __init__(self, group=None, attn_fn=None, variant: str = "hyvideo", dense_fn=None):
        self.group = group
        self._attn_fn = attn_fn
        self._dense_fn = dense_fn or _dense_shim
        self.variant = variant  # "hyvideo" | "hyvideo_i2v" (ragged text: 400 tokens -> 4 blocks) | "wan"

    def _attn(self, *a, **k):
        if self._attn_fn is None:
            from .attention import block_sparse_attention_variant
            v = self.variant
            self._attn_fn = lambda q, k_, v_, **kw: block_sparse_attention_variant(v, q, k_, v_, kw.pop("top_k"), **kw)
        return self._attn_fn(*a, **k)

    def __call__(self, attn, query, key, value, *, joint_tensor_query=None, joint_tensor_key=None,
                 joint_tensor_value=None, joint_strategy="none", top_k=0, text_amp=0.0,
                 block_neighbor_list=None, p_remain_rates=0.0, cu_seqlens_q=None, cu_seqlens_kv=None,
                 first_frame_blocks=0, dense=False, seq_len=None, **_unused):
        P, r = _group_size_rank(self.group)
        B, q_len, H, D = query.shape
        h = H // P
        joint = joint_tensor_query is not None
        if joint and joint_strategy != "rear":
            # the reference also implements "front"; Jenga's blocks only ever pass "rear"
            raise ValueError("only joint_strategy='rear' is built (attenion.py:181)")
        if joint != (joint_tensor_key is not None) or joint != (joint_tensor_value is not None):
            raise ValueError("joint_tensor_query/key/value must be given together")
        T = joint_tensor_query.shape[1] if joint else 0
        N = P * q_len
        L = _valid_rows(seq_len, N, q_len, T, dense, first_frame_blocks)
        dev, dt = query.device, query.dtype
        # receive buffers already shaped [B, N+T, h, D] so text rows are appended in place
        qkv = [torch.empty((B, N + T, h, D), dtype=dt, device=dev) for _ in range(3)]
        for buf, x in zip(qkv, (query, key, value)):
            seq_to_heads(x, self.group, out=buf[:, :N])
        if joint:
            sl = slice(r * h, (r + 1) * h)
            qkv[0][:, N:] = joint_tensor_query[:, :, sl]
            qkv[1][:, N:] = joint_tensor_key[:, :, sl]
            qkv[2][:, N:] = joint_tensor_value[:, :, sl]
        # ref :183-184 — cu_seqlens = [0, txt_len + P*q_len, S]; txt_len = cu_seqlens_q[1] - q_len.
        # Stays on the device (the reference's torch.tensor([...]) forces a host sync here).
        if cu_seqlens_q is not None:
            valid = (cu_seqlens_q[1:2].to(device=dev, dtype=torch.int32) - q_len) + N
            cu = torch.cat([torch.zeros(1, dtype=torch.int32, device=dev), valid,
                            torch.full((1,), N + T, dtype=torch.int32, device=dev)])
        else:
            cu = None
        if dense:
            out = self._dense_fn(*(x[:, :L] for x in qkv))
        else:
            # the first L rows (all N + T without seq_len); first_frame_blocks only when given, so the
            # attn_fn of every other caller sees the arguments it always saw
            ff = {"first_frame_blocks": first_frame_blocks} if first_frame_blocks else {}
            out = self._attn(*(x[:, :L + T] for x in qkv), top_k=top_k, block_size_M=128, block_size_N=128,
                             cu_seqlens_q=cu, cu_seqlens_kv=cu, text_amp=text_amp,
                             block_neighbor_list=block_neighbor_list, p_remain_rates=p_remain_rates,
                             shape_xfuse=True, text_blocks=(T + BLOCK - 1) // BLOCK if joint else 0, **ff)
        if L < N:
            full = torch.zeros((B, N, h, D), dtype=out.dtype, device=out.device)   # the pad rows stay zero
            full[:, :L] = out
            out = full
        img = heads_to_seq(out[:, :N], self.group)
        if not joint:
            return img
        txt = gather_heads(out[:, N:], self.group)
        return torch.cat([img, txt], dim=1)


class UlyssesFusedAttention:
    """Same contract as UlyssesCarvedAttention, with the exchange fused into the kernels over
    NVLink peer memory (torch symmetric memory provides the mapped pointers):

      in : jenga_ulysses_scatter stores this rank's Q/K/V image rows into every rank's
           [3, N+T, H/P, D] buffer with 16-byte peer stores — replaces three all-to-alls and their
           .contiguous() staging copies; text rows are a local head-slice copy.  The rank's H/P
           heads are processed as `groups` head sub-groups: the exchange of sub-group g+1 runs on
           a second stream UNDER the attention of sub-group g, so only the first sub-group's
           exchange is exposed.
      out: the attention kernel's epilogue stores each finished O row straight into the token
           owner's [n_loc+T, H, D] buffer (text rows into every rank's) — replaces the
           all-to-all, the all-gather and the permute copies.  The result buffer is double
           buffered across calls (no copy out): the tensor returned by call i stays valid until
           call i+2 is issued on the same stream.
    Device-side barriers (symmetric-memory signal pads) order the peer traffic: one per sub-group
    after its exchange, one per call after the attention.  The operator's opt-in switches
    (attention.QK_INT8, attention.PV_FP8) apply: a sub-group's q, k, v are quantised on the main
    stream once its exchange is complete, and the next call's exchange waits for the main stream."""

    def __init__(self, group=None, variant: str = "hyvideo", groups: int | None = None):
        self.group = group if group is not None else dist.group.WORLD
        self.variant = variant
        if groups is None:
            import os
            env = os.environ.get("JENGA_ULYSSES_GROUPS", "")
            groups = int(env) if env.isdigit() and int(env) > 0 else None   # tuning / test override
        self.groups = groups
        self._bufs = {}
        self._pad_len = {}          # result buffer -> the seq_len of its last call
        self._side = None
        self._call = 0

    def _buffers(self, N, T, h, D, n_loc, H, dtype, dev):
        import ctypes as C
        import torch.distributed._symmetric_memory as symm
        key = (N, T, h, D, n_loc, H, dtype, str(dev))
        hit = self._bufs.get(key)
        if hit is not None:
            return hit
        P = dist.get_world_size(self.group)
        try:
            symm.enable_symm_mem_for_group(self.group.group_name)
        except Exception:
            pass
        qkv = symm.empty((3, N + T, h, D), dtype=dtype, device=dev)
        h_qkv = symm.rendezvous(qkv, self.group.group_name)
        p_qkv = (C.c_uint64 * P)(*[int(x) for x in h_qkv.buffer_ptrs])
        outs = []
        for _ in range(2):
            out = symm.empty((n_loc + T, H, D), dtype=dtype, device=dev)
            h_out = symm.rendezvous(out, self.group.group_name)
            outs.append((out, h_out, (C.c_uint64 * P)(*[int(x) for x in h_out.buffer_ptrs])))
        self._bufs[key] = (qkv, h_qkv, p_qkv, outs)
        return self._bufs[key]

    @staticmethod
    def _n_groups(h: int, want: int | None, q_blocks: int | None = None) -> int:
        """Head sub-groups per rank.  Each sub-group is its own attention launch of
        (h/G) * q_blocks CTAs, one per SM at a time on the 132 SMs of an H100: a launch of only a few
        waves pays its nearly empty last wave (902 CTAs = 6.8 waves run as 7), which costs more than
        the exposed exchange saves — so sub-groups are used only while every launch stays >= 12
        waves."""
        if want:
            if h % want:
                raise ValueError(f"{h} heads per rank do not split into {want} groups")
            return want
        for g in (3, 2):
            if h % g == 0 and h >= g and (q_blocks is None or (h // g) * q_blocks >= 12 * 132):
                return g
        return 1

    def __call__(self, attn, query, key, value, *, joint_tensor_query=None, joint_tensor_key=None,
                 joint_tensor_value=None, joint_strategy="none", top_k=0, text_amp=0.0,
                 block_neighbor_list=None, p_remain_rates=0.0, cu_seqlens_q=None, cu_seqlens_kv=None,
                 first_frame_blocks=0, dense=False, seq_len=None, _hooks=None, **_unused):
        import ctypes as C
        from . import _lib
        from . import attention as A
        from ._lib import check, lib
        from .attention import _stream_ptr, block_sparse_attention_variant
        P, r = _group_size_rank(self.group)
        B, n, H, D = query.shape
        if B != 1:
            raise ValueError("the fused Ulysses path is built for batch 1 (what the pipelines run)")
        hooks = _hooks or {}
        h = H // P
        joint = joint_tensor_query is not None
        if joint and joint_strategy != "rear":
            raise ValueError("only joint_strategy='rear' is built (attenion.py:181)")
        if joint != (joint_tensor_key is not None) or joint != (joint_tensor_value is not None):
            raise ValueError("joint_tensor_query/key/value must be given together")
        T = joint_tensor_query.shape[1] if joint else 0
        N = P * n
        L = _valid_rows(seq_len, N, n, T, dense, first_frame_blocks)
        dev, dt = query.device, query.dtype
        qkv, h_qkv, p_qkv, outs = self._buffers(N, T, h, D, n, H, dt, dev)
        out, h_out, p_out = outs[self._call & 1]
        self._call += 1
        # this rank's pad rows (global rows >= L): no rank stores them, so they are zeroed whenever the
        # buffer is first used at this L
        pad0 = min(n, max(0, L - r * n))
        if self._pad_len.get(out.data_ptr(), N) != L and pad0 < n:
            out[pad0:n].zero_()
        self._pad_len[out.data_ptr()] = L
        G = self._n_groups(h, self.groups, (L + T + BLOCK - 1) // BLOCK)
        hg = h // G
        xs = [t[0] for t in (query, key, value)]
        for t in xs:
            if t.stride(2) != 1 or t.stride(1) != D or t.stride(0) != xs[0].stride(0):
                raise ValueError("q/k/v must be [1, n, H, D] views with contiguous heads and one row stride")
        a = _lib.JengaUlyssesScatterArgs()
        a.x = (C.c_void_p * 3)(*[t.data_ptr() for t in xs])
        a.x_stride_s = xs[0].stride(0)
        if joint:
            js = [t[0] for t in (joint_tensor_query, joint_tensor_key, joint_tensor_value)]
            for t in js:
                if t.stride(2) != 1 or t.stride(1) != D:
                    raise ValueError("joint tensors must be [1, T, H, D] views with contiguous heads")
            a.joint = (C.c_void_p * 3)(*[t.data_ptr() for t in js])
            a.joint_stride_s = js[0].stride(0)
        a.world, a.rank, a.heads, a.head_dim, a.n_loc, a.n_text = P, r, H, D, n, T
        a.peer_qkv_host = C.addressof(p_qkv)
        main = torch.cuda.current_stream(dev)
        if self._side is None:
            self._side = torch.cuda.Stream(device=dev)
        side = self._side if (G > 1 or hooks) else main
        events = []
        if side is not main:
            side.wait_stream(main)      # q,k,v are ready; every rank has left the previous call (its end barrier)
        with torch.cuda.stream(side), torch.cuda.device(dev):
            for g in range(G):
                if "pre_scatter" in hooks:
                    hooks["pre_scatter"](g, side)
                a.head_begin, a.head_count = g * hg, hg
                check(lib.jenga_ulysses_scatter(C.byref(a), _stream_ptr(dev)), "ulysses_scatter")
                if "post_scatter" in hooks:
                    hooks["post_scatter"](g, side)
                h_qkv.barrier(channel=0)
                if side is not main:
                    ev = torch.cuda.Event()
                    ev.record(side)
                    events.append(ev)
        if cu_seqlens_q is not None:
            valid = (cu_seqlens_q[1:2].to(device=dev, dtype=torch.int32) - n) + N
            cu = torch.cat([torch.zeros(1, dtype=torch.int32, device=dev), valid,
                            torch.full((1,), N + T, dtype=torch.int32, device=dev)])
        else:
            cu = None
        for g in range(G):
            if side is not main:
                main.wait_event(events[g])
            sl = slice(g * hg, (g + 1) * hg)
            sp = dict(world=P, rank=r, heads_total=H, rows=n, peers=p_out, head_base=r * h + g * hg)
            q, k, v = (x[None, :L + T, sl] for x in qkv)       # all N + T rows without seq_len
            if dense:
                # flash_attn_shim._dense's launch, with the peer-store epilogue instead of `out`
                v8, qk8 = A.quantize_operands(q, k, v, A.PV_FP8, A.QK_INT8)
                A._launch(q, k, v, None, 0, (L + BLOCK - 1) // BLOCK, D ** -0.5, 0.0, 1 << 30, L, L, L, None,
                          None, q.dtype, sp_out=sp, v_fp8=v8, qk_int8=qk8)
            else:
                block_sparse_attention_variant(self.variant, q, k, v, top_k, cu_seqlens_q=cu, cu_seqlens_kv=cu,
                                               text_blocks=(T + BLOCK - 1) // BLOCK, text_amp=text_amp,
                                               block_neighbor_list=block_neighbor_list,
                                               p_remain_rates=p_remain_rates, first_frame_blocks=first_frame_blocks,
                                               sp_out=sp)
            if "post_attention" in hooks:
                # per-group completion across ranks, so the caller may drain this group's heads
                h_out.barrier(channel=0)
                hooks["post_attention"](g, main, out, hg)
        if "post_attention" not in hooks:
            h_out.barrier(channel=0)
        return out[None]

    def plan(self, heads_per_rank: int, tokens: int | None = None) -> tuple[int, int]:
        """(groups, heads per group) this object will use for `heads_per_rank` heads over `tokens`
        (global sequence length incl. text) tokens."""
        G = self._n_groups(heads_per_rank, self.groups, None if tokens is None else (tokens + BLOCK - 1) // BLOCK)
        return G, heads_per_rank // G


class HostPipelinedUlysses:
    """Sequence-parallel AttenCarve for callers whose per-rank activations live in PINNED HOST
    memory: `hq, hk, hv` [1, n_loc+T, H, D] (this rank's token slice + the replicated text rows,
    all heads) in, `hout` [1, n_loc+T, H, D] out.  Four streams per rank, pipelined by head
    sub-group (the operator is independent per head, SURVEY §8e):

        copy-in : H2D of sub-group g+1 (strided 2-D copies)   — also runs ahead into the NEXT call
        side    : peer-store exchange of sub-group g (jenga_ulysses_scatter) + device barrier
        main    : selection + carved attention of sub-group g (epilogue peer-stores O rows)
        copy-out: D2H of sub-group g-1

    Results are bit-identical to UlyssesFusedAttention on device-resident tensors."""

    def __init__(self, n_loc: int, T: int, H: int, D: int = 128, dtype=torch.bfloat16, device="cuda",
                 fused: UlyssesFusedAttention | None = None):
        from ._lib import check, lib  # noqa: F401
        self.fused = fused or UlyssesFusedAttention()
        self.dev = torch.device(device)
        self.n, self.T, self.H, self.D = n_loc, T, H, D
        P = dist.get_world_size(self.fused.group)
        self.P, self.h = P, H // P
        self.G, self.hg = self.fused.plan(self.h, P * n_loc + T)
        mk = lambda: torch.empty((1, n_loc + T, H, D), dtype=dtype, device=self.dev)  # noqa: E731
        self.dq, self.dk, self.dv = mk(), mk(), mk()
        self.s_in = torch.cuda.Stream(self.dev)
        self.s_out = torch.cuda.Stream(self.dev)
        self.ev_in = [torch.cuda.Event() for _ in range(self.G)]
        self.ev_scattered = [None] * self.G
        self._ev_out = [None, None]     # copy-out completion per result buffer (the result is double-buffered)
        self._first = True

    def finish(self) -> None:
        """Makes the current stream wait for every copy-out issued so far (call after a run of
        `__call__(..., wait=False)` steps, before the host reads `hout`)."""
        torch.cuda.current_stream(self.dev).wait_stream(self.s_out)

    def __call__(self, hq, hk, hv, hout, wait: bool = True, **kw):
        """wait=False lets consecutive calls overlap: copy-in of step i+1 runs under the attention of
        step i and the copy-out of step i under step i+1; call finish() before reading `hout`."""
        from .host_pipeline import _copy2d
        n, T, H, D, P, h, G, hg = self.n, self.T, self.H, self.D, self.P, self.h, self.G, self.hg
        for t in (hq, hk, hv, hout):
            if tuple(t.shape) != (1, n + T, H, D) or not t.is_contiguous() or not t.is_pinned():
                raise ValueError("host tensors must be pinned, contiguous [1, n_loc+T, H, D]")
        es = hq.element_size()
        pitch, width, rows = h * D * es, hg * D * es, (n + T) * P   # rows = (token, destination rank)
        main = torch.cuda.current_stream(self.dev)
        if self._first:
            self.s_in.wait_stream(main)     # staging buffers were allocated on `main`
            self._first = False
        par = self.fused._call & 1          # which of the two result buffers this call fills
        if self._ev_out[par] is not None:
            main.wait_event(self._ev_out[par])   # its previous contents have been copied out
        for g in range(G):
            if self.ev_scattered[g] is not None:
                self.s_in.wait_event(self.ev_scattered[g])   # the previous call has consumed this staging slice
            off = g * hg * D * es
            if G == 1:      # the whole slice is one contiguous copy
                with torch.cuda.stream(self.s_in):
                    for dst, src in ((self.dq, hq), (self.dk, hk), (self.dv, hv)):
                        dst.copy_(src, non_blocking=True)
            else:
                for dst, src in ((self.dq, hq), (self.dk, hk), (self.dv, hv)):
                    _copy2d(dst.data_ptr() + off, pitch, src.data_ptr() + off, pitch, width, rows, 0, self.s_in)
            self.ev_in[g].record(self.s_in)

        def pre_scatter(g, side):
            side.wait_event(self.ev_in[g])

        def post_scatter(g, side):
            ev = torch.cuda.Event()
            ev.record(side)
            self.ev_scattered[g] = ev

        def post_attention(g, main_s, out, hg_):
            ev = torch.cuda.Event()
            ev.record(main_s)
            self.s_out.wait_event(ev)
            off = g * hg * D * es
            if G == 1:
                with torch.cuda.stream(self.s_out):
                    hout.copy_(out.view(hout.shape), non_blocking=True)
            else:
                _copy2d(hout.data_ptr() + off, pitch, out.data_ptr() + off, pitch, width, rows, 1, self.s_out)

        self.fused(None, self.dq[:, :n], self.dk[:, :n], self.dv[:, :n],
                   joint_tensor_query=self.dq[:, n:] if T else None, joint_tensor_key=self.dk[:, n:] if T else None,
                   joint_tensor_value=self.dv[:, n:] if T else None, joint_strategy="rear" if T else "none",
                   _hooks=dict(pre_scatter=pre_scatter, post_scatter=post_scatter, post_attention=post_attention), **kw)
        ev = torch.cuda.Event()
        ev.record(self.s_out)
        self._ev_out[par] = ev
        if wait:
            main.wait_stream(self.s_out)
        return hout


def my_parallel_attention(hybrid_seq_parallel_attn, q, k, v, img_q_len, img_kv_len, cu_seqlens_q,
                          cu_seqlens_kv, top_k=int(10e7), text_amp=0.0, block_neighbor_list=None,
                          p_remain_rates=0.0):
    """attenion.py:159-195, verbatim contract: q,k,v are img||txt per rank; returns [B, s, H*D]."""
    attn = hybrid_seq_parallel_attn(
        None, q[:, :img_q_len], k[:, :img_kv_len], v[:, :img_kv_len],
        joint_tensor_query=q[:, img_q_len:], joint_tensor_key=k[:, img_kv_len:],
        joint_tensor_value=v[:, img_kv_len:], joint_strategy="rear", top_k=top_k,
        cu_seqlens_q=cu_seqlens_q, cu_seqlens_kv=cu_seqlens_kv, text_amp=text_amp,
        block_neighbor_list=block_neighbor_list, p_remain_rates=p_remain_rates)
    b, s, a, d = attn.shape
    return attn.reshape(b, s, -1)


# --------------------------------------------------------------------------------------------
# bench.py helpers (N > 1): every rank builds ITS slice of the same global layer input
# --------------------------------------------------------------------------------------------
def bench_setup(wl, build_inputs, dev, rank, world):
    full = build_inputs(wl, dev)  # identical seeds on every rank -> identical global tensors
    n_img = full["n_img"]
    assert n_img % world == 0, "image tokens must divide by the SP degree (jenga_hyvideo_multigpu.py:168-171)"
    n_loc = n_img // world
    sl = slice(rank * n_loc, (rank + 1) * n_loc)
    q = torch.cat([full["q"][:, sl], full["q"][:, n_img:]], dim=1).contiguous()
    k = torch.cat([full["k"][:, sl], full["k"][:, n_img:]], dim=1).contiguous()
    v = torch.cat([full["v"][:, sl], full["v"][:, n_img:]], dim=1).contiguous()
    # local cu_seqlens as get_cu_seqlens would build them from local shapes (attenion.py:34-57)
    cu = torch.tensor([0, n_loc + wl["text_valid"], n_loc + wl["text_tokens"]], dtype=torch.int32, device=dev)
    top_k = world * int((1 - wl["drop"]) * (n_loc // BLOCK))  # models_mul…:242,249-251
    inp = dict(full)
    del full
    inp.update(q=None, k=None, v=None, top_k=top_k)
    torch.cuda.empty_cache()
    import os
    import sys
    fused = os.environ.get("JENGA_ULYSSES", "fused") != "nccl"
    st = dict(q=q, k=k, v=v, cu=cu, n_loc=n_loc, top_k=top_k, inp=inp, world=world, rank=rank)
    if fused:
        # Both modes are GPU paths of this library.  The fused one needs peer-mapped symmetric
        # memory; if the rendezvous is refused on this box (no P2P), every rank agrees to use NCCL.
        ok = 1
        try:
            st["sp"] = UlyssesFusedAttention(variant=wl["variant"])
            bench_step(wl, st)
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            ok = 0
            print(f"[bench] rank {rank}: fused Ulysses unavailable ({type(e).__name__}: {e}); using NCCL",
                  file=sys.stderr)
        t = torch.tensor([ok], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        fused = bool(t.item())
    if not fused:
        st["sp"] = UlyssesCarvedAttention(variant=wl["variant"])
    st["mode"] = "fused peer stores" if fused else "nccl all-to-all"
    return st


def bench_step(wl, st):
    return my_parallel_attention(st["sp"], st["q"], st["k"], st["v"], st["n_loc"], st["n_loc"], st["cu"],
                                 st["cu"], top_k=st["top_k"], text_amp=wl["text_amp"],
                                 block_neighbor_list=st["inp"]["nbr"], p_remain_rates=wl["p_remain"])


def bench_flops(wl, st, algorithmic_flops):
    """Sum over ranks of the live tiles of each rank's head group."""
    from .attention import block_sparse_attention_variant
    captured = {}

    def attn_fn(q, k, v, **kw):
        kw.pop("shape_xfuse", None)
        o, bits = block_sparse_attention_variant(wl["variant"], q, k, v, kw.pop("top_k"), shape_xfuse=True,
                                                 return_mask_bits=True, **kw)
        captured["bits"] = bits
        captured["heads"] = q.shape[2]
        return o

    sp = UlyssesCarvedAttention(attn_fn=attn_fn, variant=wl["variant"])
    my_parallel_attention(sp, st["q"], st["k"], st["v"], st["n_loc"], st["n_loc"], st["cu"], st["cu"],
                          top_k=st["top_k"], text_amp=wl["text_amp"], block_neighbor_list=st["inp"]["nbr"],
                          p_remain_rates=wl["p_remain"])
    inp = dict(st["inp"])
    inp["heads"] = captured["heads"]
    flops, pop = algorithmic_flops(wl, inp, captured["bits"])
    t = torch.tensor([float(flops), float(pop)], dtype=torch.float64, device=st["q"].device)
    dist.all_reduce(t)
    return int(t[0].item()), int(t[1].item())
