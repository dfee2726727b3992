"""Tensor-parallel forward for the single-sample case (BASELINE config 4): one sample's transformer forward split over the
GPUs of one node. The reference has no tensor parallelism (SURVEY.md 2c); this follows SURVEY.md 8e:

  * attention: heads split (q/k/v_proj column-parallel, attn_out row-parallel); MLP: ff split (ff_proj/up_proj
    column-parallel, ff_out row-parallel); LM head: vocabulary rows split (and the VQ-codebook window split separately);
  * the two row-parallel GEMMs per layer produce fp32 PARTIAL sums (MMDP_EPI_F32). What follows them - the cross-rank sum,
    the residual add, the NEXT RMSNorm and the distribution of its output to all ranks - is one kernel per rank over NVLink
    peer memory: the GEMM's epilogue PUSHES every fp32 partial row into the receive buffer of the rank that owns it
    (`mmdp_gemm_f32_scatter`: the reduce-scatter is fused into the GEMM and overlaps its main loop), then
    `mmdp_tp_reduce_norm` (csrc/tp_collective.cu) sums the rows a rank owns in fixed rank order, applies the single-GPU
    rounding points `x = bf16(bf16(sum) + x)` and the norm, and stores the bf16 result into every rank's activation buffer
    (the all-gather). The residual stream is row-sharded (M / TP rows per rank), the normalised activations are replicated;
    0.75x the bytes of an fp32 all-reduce, all of them NVLink writes, and no separate residual / RMSNorm launches;
  * every rank gathers the logits slices it needs (NCCL all_gather, once per forward) and runs the SAME sampling kernels on
    the same noise (identical generator seeds), so the id sequence stays in sync without broadcasts.

`collective="nccl"` keeps round 1's formulation (fp32 `dist.all_reduce` + `mmdp_resid_add_f32` + `mmdp_rmsnorm` between the
kernels) as the measured baseline of the peer-memory path (bench.py --tp --tp-collective nccl).
Buffers shared between the ranks are plain cudaMalloc allocations exported with CUDA IPC (`mmdp_ipc_export/import`); the
handles travel through `dist.all_gather_object`.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from . import _lib
from ._lib import EPI_F32, EPI_PLAIN, EPI_SWIGLU, check, lib, ptr, stream_ptr
from .model import ModelOutput, check_supported_config, rope_tables


def shard_state_dict(sd: Dict[str, torch.Tensor], n_layers: int, n_heads: int, rank: int, tp: int, vq_col0: int,
                     vq_cols: int) -> Dict[str, torch.Tensor]:
    """Slices a full HF state dict (names of SURVEY.md 8b) into rank `rank`'s tensor-parallel shard. Pure tensor slicing
    (device agnostic) so it is unit-tested on the CPU."""
    g = lambda n: sd["model.transformer." + n] if ("model.transformer." + n) in sd else sd[n]
    out = {"wte": g("wte.weight"), "ln_f": g("ln_f.weight")}
    head = g("ff_out.weight")
    V, d = head.shape
    if n_heads % tp or V % tp or vq_cols % tp:
        raise ValueError(f"tp={tp} must divide n_heads={n_heads}, vocab rows={V} and the codebook window={vq_cols}")
    da = (n_heads // tp) * 128
    out["head"] = head[rank * (V // tp):(rank + 1) * (V // tp)]
    c = vq_cols // tp
    out["head_vq"] = head[vq_col0 + rank * c: vq_col0 + (rank + 1) * c]
    for i in range(n_layers):
        p = f"blocks.{i}."
        sl = slice(rank * da, (rank + 1) * da)
        out[p + "wqkv"] = torch.cat([g(p + "q_proj.weight")[sl], g(p + "k_proj.weight")[sl], g(p + "v_proj.weight")[sl]], dim=0)
        out[p + "wo"] = g(p + "attn_out.weight")[:, sl]
        ffp, up = g(p + "ff_proj.weight"), g(p + "up_proj.weight")
        ff = ffp.shape[0]
        if (ff // tp) % 128:
            raise ValueError("mlp_hidden / tp must be a multiple of 128 (SwiGLU tile interleave)")
        fs = slice(rank * (ff // tp), (rank + 1) * (ff // tp))
        g1, u1 = ffp[fs], up[fs]
        nb = g1.shape[0] // 128
        w13 = torch.stack([g1.reshape(nb, 128, d), u1.reshape(nb, 128, d)], dim=1).reshape(2 * nb * 128, d)
        out[p + "w13"] = w13
        out[p + "w2"] = g(p + "ff_out.weight")[:, fs]
        out[p + "attn_norm"] = g(p + "attn_norm.weight")
        out[p + "ff_norm"] = g(p + "ff_norm.weight")
    return out


def rows_per_rank(M: int, tp: int) -> int:
    return (M + tp - 1) // tp


def row_partition(M: int, tp: int, rank: int):
    """Rows of the residual stream rank `rank` owns: [rank * R, min((rank + 1) * R, M)) with R = ceil(M / tp) - the owner of a
    row is row // R, which the GEMM's scatter epilogue evaluates per row. Returns (first row, count); the count of the last
    ranks can be 0 for tiny M (rejected by the caller: every rank has to take part in the collective)."""
    R = rows_per_rank(M, tp)
    r0 = rank * R
    return r0, max(0, min(R, M - r0))


def chunk_split(M: int) -> List[int]:
    """Row chunks of the pipelined tensor-parallel forward: [M] for short sequences, else two chunks, the first a multiple of
    256 rows (whole CTA-pair GEMM tiles) closest to M / 2 from above. With two chunks the attn_out / MLP part of a layer runs as
    two independent chains on two streams: one chunk's NVLink traffic overlaps the other chunk's GEMMs (csrc/api.cu,
    mmdp_tp_forward)."""
    if M < 1024:
        return [M]
    r0 = (M // 2 + 255) // 256 * 256
    return [r0, M - r0]


class _DeviceArray:
    """Zero-copy torch view of a raw device allocation (a cudaMalloc made by libmmdp for IPC export)."""

    def __init__(self, ptr_value: int, numel: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (numel,), "typestr": typestr, "data": (int(ptr_value), False), "version": 3}


class _SharedBuffer:
    """One buffer per rank, visible to all ranks of the node: `ptrs[r]` is rank r's allocation mapped into this process."""

    def __init__(self, nbytes: int, rank: int, world: int, group):
        self.rank, self.world = rank, world
        own = C.c_void_p()
        check(lib.mmdp_tp_alloc(nbytes, C.byref(own)))
        self.own = own.value
        handle = (C.c_uint8 * 64)()
        check(lib.mmdp_ipc_export(self.own, handle))
        handles: List[Optional[bytes]] = [None] * world
        dist.all_gather_object(handles, bytes(handle), group=group)
        self.ptrs: List[int] = []
        self._imported: List[int] = []
        for r in range(world):
            if r == rank:
                self.ptrs.append(self.own)
                continue
            p = C.c_void_p()
            buf = (C.c_uint8 * 64).from_buffer_copy(handles[r])
            check(lib.mmdp_ipc_import(buf, C.byref(p)))
            self.ptrs.append(p.value)
            self._imported.append(p.value)
        self.array = (C.c_void_p * world)(*self.ptrs)   # host array of device pointers for the C ABI

    def close(self):
        for p in self._imported:
            lib.mmdp_ipc_close(p)
        self._imported = []
        if self.own:
            lib.mmdp_tp_free(self.own)
            self.own = None


class TensorParallelLLaDA:
    """Same call contract as model.LLaDAForMultiModalGeneration (`forward_rows`, `__call__`), one rank of a TP group."""

    def __init__(self, config, state_dict: Dict[str, torch.Tensor], tp_rank: int, tp_size: int, group=None,
                 max_seq_len: Optional[int] = None, max_batch: int = 1, device: str = "cuda:0", text_vocab_size: int = 126356,
                 codebook_size: int = 8192, collective: str = "p2p", chunks: Optional[int] = None):
        if not torch.cuda.is_available():
            raise _lib.MmdpError("mmada_parallel_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        if collective not in ("p2p", "nccl"):
            raise ValueError("collective must be 'p2p' (NVLink peer-memory kernel) or 'nccl' (all-reduce baseline)")
        self.config, self.group, self.rank, self.tp = config, group, tp_rank, tp_size
        self.collective = collective if tp_size > 1 else "nccl"
        if chunks is None:
            # one chunk by default: two half-size chains on two streams halve the GEMMs and double the launches, which has cost more
            # than the NVLink time they hide. The schedule stays available (chunks=2, bitwise identical results).
            chunks = 1
        if chunks not in (1, 2):
            raise ValueError("chunks must be 1 or 2")
        self.chunks = chunks
        self._alloc_chunks = 2  # buffers for both schedules (chunk 1: half of the workspace rows)
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        g = lambda k, dflt=None: getattr(config, k, dflt)
        self.d_model, self.n_heads, self.n_layers = int(g("d_model")), int(g("n_heads")), int(g("n_layers"))
        self.ff = int(g("mlp_hidden_size") or g("mlp_ratio", 4) * self.d_model)
        self.vocab_rows = int(g("embedding_size") or g("vocab_size"))
        self.rms_eps = float(g("rms_norm_eps", 1e-5))
        check_supported_config(config, self.n_heads)
        self.h_local = self.n_heads // tp_size
        self.d_attn = self.h_local * 128
        if self.d_attn % 256:
            raise ValueError("n_heads / tp must be even (the fused QKV+RoPE epilogue works on 2-head tiles)")
        self.ff_local = self.ff // tp_size
        self.v_local = self.vocab_rows // tp_size
        self.vq_col0, self.vq_cols = text_vocab_size, codebook_size
        self.c_local = codebook_size // tp_size
        self.max_seq_len = int(max_seq_len or g("max_sequence_length", 4096))
        self.max_batch = max_batch
        sh = shard_state_dict(state_dict, self.n_layers, self.n_heads, tp_rank, tp_size, text_vocab_size, codebook_size)
        self.w = {k: v.detach().to(device=self.device, dtype=torch.bfloat16).contiguous() for k, v in sh.items()}
        cos, sin = rope_tables(128, float(g("rope_theta", 10000.0)), self.max_seq_len)
        self.cos, self.sin = cos.to(self.device), sin.to(self.device)
        M, d, bf = self.max_batch * self.max_seq_len, self.d_model, dict(dtype=torch.bfloat16, device=self.device)
        self.Mmax = M
        self.q = torch.empty((M, self.d_attn), **bf)
        self.k = torch.empty((M, self.d_attn), **bf)
        self.att = torch.empty((M, self.d_attn), **bf)
        self.h = torch.empty((M, self.ff_local), **bf)
        self.vt = None
        self._vt_key = None
        if self.collective == "p2p":
            if M < tp_size:
                raise ValueError("the workspace must hold at least one row per rank")
            # per row chunk (see chunk_split): receive buffers [tp][R][d] fp32 (slot r <- rank r's partial rows for the rows this
            # rank owns), used alternately; flags; this rank's rows of the residual stream. Chunk 0 is sized for the whole
            # workspace (a short sequence runs as one chunk), chunk 1 for half of it.
            self._chunk_state = []
            for ci in range(self._alloc_chunks):
                rows = M if ci == 0 else (M + 1) // 2          # chunk 1 never holds more than half of the rows (chunk_split)
                R = rows_per_rank(rows, tp_size)
                st = {"recv": [_SharedBuffer(tp_size * R * d * 4, tp_rank, tp_size, group) for _ in range(2)],
                      "flags": _SharedBuffer(2 * 8 * 4, tp_rank, tp_size, group),
                      "x": torch.empty((R, d), **bf), "done": torch.zeros(1, dtype=torch.int32, device=self.device)}
                self._chunk_state.append(st)
            self._xn = _SharedBuffer(M * d * 2, tp_rank, tp_size, group)
            self.xn = torch.as_tensor(_DeviceArray(self._xn.own, M * d, "<u2"), device=self.device).view(torch.bfloat16).view(M, d)
            self.x = self._chunk_state[0]["x"]
            self._epoch = 0
            torch.cuda.synchronize()
            dist.barrier(group=group)  # every rank has mapped every buffer before the first peer access
        else:
            self.x = torch.empty((M, d), **bf)
            self.xn = torch.empty((M, d), **bf)
            self.part = torch.empty((M, d), dtype=torch.float32, device=self.device)

    def __del__(self):
        shared = [getattr(self, "_xn", None)]
        for st in getattr(self, "_chunk_state", []):
            shared += st["recv"] + [st["flags"]]
        for b in shared:
            if b is not None:
                try:
                    b.close()
                except Exception:
                    pass

    def eval(self):
        return self

    def _allreduce(self, t: torch.Tensor):
        if self.tp > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)

    def _gather_cols(self, local: torch.Tensor, out: torch.Tensor):
        """local [n, c] on every rank -> out [n, tp*c] (rank r's block at columns r*c)."""
        if self.tp == 1:
            out.copy_(local)
            return
        n, c = local.shape
        buf = torch.empty((self.tp, n, c), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(buf, local.contiguous(), group=self.group)
        out.view(n, self.tp, c).copy_(buf.permute(1, 0, 2))

    # ------------------------------------------------------------------------------------------------------------------
    def _layers_nccl(self, B: int, L: int, M: int, Lpad: int):
        """Round 1's formulation, kept as the measured baseline (`collective="nccl"`): fp32 partial sums stored locally,
        `dist.all_reduce` between the kernels, then the residual add and the RMSNorm as separate launches."""
        d, s, w = self.d_model, stream_ptr(), self.w
        scale = 1.0 / math.sqrt(128.0)
        x, xn = self.x, self.xn
        for i in range(self.n_layers):
            p = f"blocks.{i}."
            check(lib.mmdp_rmsnorm(ptr(x), d, None, ptr(w[p + "attn_norm"]), ptr(xn), d, M, d, self.rms_eps, s))
            check(lib.mmdp_qkv_rope_tp(ptr(xn), d, ptr(w[p + "wqkv"]), M, d, self.h_local, L, Lpad, ptr(self.cos), ptr(self.sin),
                                       ptr(self.q), ptr(self.k), ptr(self.vt), s))
            check(lib.mmdp_attention(ptr(self.q), ptr(self.k), ptr(self.vt), ptr(self.att), B, self.h_local, L, Lpad, scale, s))
            check(lib.mmdp_gemm_bf16(EPI_F32, ptr(self.att), self.d_attn, ptr(w[p + "wo"]), self.d_attn, M, d, self.d_attn,
                                     ptr(self.part), d, None, 0, s))
            self._allreduce(self.part[:M])
            check(lib.mmdp_resid_add_f32(ptr(x), d, ptr(self.part), d, M, d, s))
            check(lib.mmdp_rmsnorm(ptr(x), d, None, ptr(w[p + "ff_norm"]), ptr(xn), d, M, d, self.rms_eps, s))
            check(lib.mmdp_gemm_bf16(EPI_SWIGLU, ptr(xn), d, ptr(w[p + "w13"]), d, M, 2 * self.ff_local, d, ptr(self.h),
                                     self.ff_local, None, 0, s))
            check(lib.mmdp_gemm_bf16(EPI_F32, ptr(self.h), self.ff_local, ptr(w[p + "w2"]), self.ff_local, M, d, self.ff_local,
                                     ptr(self.part), d, None, 0, s))
            self._allreduce(self.part[:M])
            check(lib.mmdp_resid_add_f32(ptr(x), d, ptr(self.part), d, M, d, s))

    def _native_ctx(self, B: int, L: int):
        """The C-side description of this rank (mmdp_tp_ctx): built once per (B, L) - the V^T buffer depends on it."""
        key = (B, L)
        if getattr(self, "_ctx_key", None) == key:
            return self._ctx
        w = self.w
        layers = (_lib.TpLayer * self.n_layers)()
        for i in range(self.n_layers):
            p = f"blocks.{i}."
            for name, t in (("wqkv", w[p + "wqkv"]), ("wo", w[p + "wo"]), ("w13", w[p + "w13"]), ("w2", w[p + "w2"]),
                            ("attn_norm", w[p + "attn_norm"]), ("ff_norm", w[p + "ff_norm"])):
                setattr(layers[i], name, t.data_ptr())
        c = _lib.TpCtx()
        c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = self.d_model, self.h_local, self.ff_local, self.n_layers, self.tp, self.rank
        c.rms_eps = self.rms_eps
        c.layers = layers
        c.wte, c.ln_f, c.vocab = w["wte"].data_ptr(), w["ln_f"].data_ptr(), w["wte"].shape[0]
        c.cos_tab, c.sin_tab = self.cos.data_ptr(), self.sin.data_ptr()
        c.q, c.k, c.att, c.h, c.vt = self.q.data_ptr(), self.k.data_ptr(), self.att.data_ptr(), self.h.data_ptr(), self.vt.data_ptr()
        c.xn = C.cast(self._xn.array, C.POINTER(C.c_void_p))
        split = chunk_split(B * L) if self.chunks == 2 else [B * L]
        c.n_chunks = len(split)
        c.chunk_rows0 = split[0]
        for ci in range(len(split)):
            st = self._chunk_state[ci]
            c.chunk[ci].x_shard = st["x"].data_ptr()
            c.chunk[ci].recv[0] = C.cast(st["recv"][0].array, C.POINTER(C.c_void_p))
            c.chunk[ci].recv[1] = C.cast(st["recv"][1].array, C.POINTER(C.c_void_p))
            c.chunk[ci].flags = C.cast(st["flags"].array, C.POINTER(C.c_void_p))
            c.chunk[ci].done_counter = st["done"].data_ptr()
        self._ctx, self._ctx_layers, self._ctx_key = c, layers, key   # (keep the layer array alive)
        return c

    def _final_norm(self, ids: torch.Tensor) -> torch.Tensor:
        """Runs embedding + all blocks; returns ln_f(x) for ALL rows [M, d] (p2p) or the raw residual stream x (nccl)."""
        B, L = ids.shape
        M, d, s = B * L, self.d_model, stream_ptr()
        if M > self.Mmax:
            raise _lib.MmdpError("TensorParallelLLaDA: batch x length exceeds the workspace")
        Lpad = (L + 7) // 8 * 8
        if self._vt_key != (B, Lpad, L):
            self.vt = torch.zeros((B, self.h_local, 128, Lpad), dtype=torch.bfloat16, device=self.device)
            self._vt_key = (B, Lpad, L)
        wte = self.w["wte"]
        if self.collective == "p2p":
            for rows in (chunk_split(M) if self.chunks == 2 else [M]):
                if row_partition(rows, self.tp, self.tp - 1)[1] < 1:
                    raise _lib.MmdpError(f"TensorParallelLLaDA: {rows} rows cannot be split over {self.tp} ranks with at least one row each")
            # the whole body is one native call (a Python loop of ~10 launches per layer left a TP=8 rank CPU-bound)
            out = C.c_uint32(0)
            check(lib.mmdp_tp_forward(C.byref(self._native_ctx(B, L)), ptr(ids), B, L, self._epoch, C.byref(out), s))
            self._epoch = int(out.value)
            return self.xn
        check(lib.mmdp_embed(ptr(ids), ptr(wte), ptr(self.x), M, d, wte.shape[0], s))
        self._layers_nccl(B, L, M, Lpad)
        return self.x

    @torch.no_grad()
    def forward_rows(self, ids: torch.Tensor, rows_a: Optional[torch.Tensor] = None, rows_b: Optional[torch.Tensor] = None,
                     col0_b: int = 0, ncols_b: int = 0, out_a: Optional[torch.Tensor] = None, out_b: Optional[torch.Tensor] = None):
        hid = self._final_norm(ids.contiguous())
        d, s, w = self.d_model, stream_ptr(), self.w

        def rows_normed(rows):
            n = rows.numel()
            if self.collective == "p2p":
                return hid.index_select(0, rows.long())                    # already ln_f(x): the last collective used ln_f's weight
            xr = torch.empty((n, d), dtype=torch.bfloat16, device=self.device)
            check(lib.mmdp_rmsnorm(ptr(hid), d, ptr(rows), ptr(w["ln_f"]), ptr(xr), d, n, d, self.rms_eps, s))
            return xr

        ra = rb = None
        if rows_a is not None and rows_a.numel():
            n = rows_a.numel()
            loc = _lib.gemm_bf16(rows_normed(rows_a), w["head"], EPI_PLAIN)
            ra = out_a if out_a is not None else torch.empty((n, self.vocab_rows), dtype=torch.bfloat16, device=self.device)
            self._gather_cols(loc, ra)
        if rows_b is not None and rows_b.numel():
            if col0_b != self.vq_col0 or ncols_b != self.vq_cols:
                raise _lib.MmdpError("TensorParallelLLaDA: the column window must be the VQ codebook window given at construction")
            n = rows_b.numel()
            loc = _lib.gemm_bf16(rows_normed(rows_b), w["head_vq"], EPI_PLAIN)
            rb = out_b if out_b is not None else torch.empty((n, ncols_b), dtype=torch.bfloat16, device=self.device)
            self._gather_cols(loc, rb)
        return ra, rb

    @torch.no_grad()
    def forward(self, input_ids=None, infer: bool = True, use_cache: bool = False, **_) -> ModelOutput:
        ids = input_ids.to(device=self.device, dtype=torch.int64)
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        B, L = ids.shape
        rows = torch.arange(B * L, dtype=torch.int32, device=self.device)
        logits, _ = self.forward_rows(ids.contiguous(), rows_a=rows)
        return ModelOutput(logits=logits.view(B, L, self.vocab_rows))

    __call__ = forward
