"""Tensor-parallel forward for the single-sample case (BASELINE config 4): one sample's transformer forward split over the
GPUs of one node. The reference has no tensor parallelism (SURVEY.md 2c); this follows SURVEY.md 8e:

  * attention: heads split (q/k/v_proj column-parallel, attn_out row-parallel; with grouped-query or multi-query attention each
    rank computes the kv heads its query heads read, see kv_shard); MLP: ff split (ff_proj/up_proj
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

`precision="fp8"` runs the four block linears in e4m3 as the single-GPU FP8 context does (DESIGN §3 "FP8 under tensor
parallel"): every weight is quantised whole (one scale per row over the full K) and then sliced (shard_state_dict_fp8), the
reduce before a column-parallel linear broadcasts e4m3 rows and their 1 x 128 group scales (`mmdp_tp_reduce_norm_fp8`), att and
h are quantised locally before the row-parallel FP8 GEMMs that push fp32 partial rows (`mmdp_gemm_fp8_f32_scatter`), and ln_f
after the last layer stays bf16 for the LM head.

Packed batches (`forward_rows_packed`, the call `generators.batch.generate_ti2ti_batch` makes) lay several sequences end to end
in one forward, each computed as if it were alone, exactly as the single-GPU model's packed forward does (DESIGN §3 "Packed
batches under tensor parallel"): only the QKV epilogue, the attention launch and the V^T layout see the sequences; row ownership,
the scatter GEMMs, the reduces and the row chunks work on the packed rows. `max_batch = N` sizes every per-rank work buffer for N
full-length sequences: q, k, att, h, xn (and in FP8 the e4m3 copy xq and a8) and the receive buffers (2 per chunk, fp32 rows of
this rank's share) all grow linearly with N.

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


def kv_shard(n_heads: int, n_kv_heads: int, rank: int, tp: int):
    """The kv heads rank `rank` of `tp` computes: (first kv head, count). Rank r owns query heads [r H / tp, (r + 1) H / tp), and
    query head h reads kv head h // (H / Hkv).
      * tp divides Hkv: rank r owns kv heads [r Hkv / tp, (r + 1) Hkv / tp), exactly those its query heads read;
      * Hkv divides tp (multi-query attention included): rank r computes the one kv head r Hkv // tp that all its query heads
        read; that kv head is computed on tp / Hkv ranks.
    Any other (tp, Hkv) pair would split one rank's query heads over kv heads owned by different ranks: ValueError."""
    if n_kv_heads % tp == 0:
        return rank * (n_kv_heads // tp), n_kv_heads // tp
    if tp % n_kv_heads == 0:
        return rank * n_kv_heads // tp, 1
    raise ValueError(f"tp={tp} and n_kv_heads={n_kv_heads}: one of the two must divide the other (each rank computes whole kv heads "
                     "for its query heads)")


def shard_state_dict(sd: Dict[str, torch.Tensor], n_layers: int, n_heads: int, rank: int, tp: int, vq_col0: int,
                     vq_cols: int, *, n_kv_heads: Optional[int] = None, qkv_bias: bool = False) -> Dict[str, torch.Tensor]:
    """Slices a full HF state dict (names of SURVEY.md 8b) into rank `rank`'s tensor-parallel shard. Pure tensor slicing
    (device agnostic) so it is unit-tested on the CPU. n_kv_heads (None: n_heads) and the kv heads of the shard follow kv_shard;
    `blocks.i.wqkv` holds the q rows of the local heads, then the k rows and the v rows of the local kv heads, and with qkv_bias
    `blocks.i.bqkv` the matching slices of the q / k / v biases."""
    g = lambda n: sd["model.transformer." + n] if ("model.transformer." + n) in sd else sd[n]
    out = {"wte": g("wte.weight"), "ln_f": g("ln_f.weight")}
    head = g("ff_out.weight")
    V, d = head.shape
    if n_heads % tp or V % tp or vq_cols % tp:
        raise ValueError(f"tp={tp} must divide n_heads={n_heads}, vocab rows={V} and the codebook window={vq_cols}")
    da = (n_heads // tp) * 128
    kv0, n_kv_local = kv_shard(n_heads, n_kv_heads or n_heads, rank, tp)
    kv = slice(kv0 * 128, (kv0 + n_kv_local) * 128)
    out["head"] = head[rank * (V // tp):(rank + 1) * (V // tp)]
    c = vq_cols // tp
    out["head_vq"] = head[vq_col0 + rank * c: vq_col0 + (rank + 1) * c]
    for i in range(n_layers):
        p = f"blocks.{i}."
        sl = slice(rank * da, (rank + 1) * da)
        out[p + "wqkv"] = torch.cat([g(p + "q_proj.weight")[sl], g(p + "k_proj.weight")[kv], g(p + "v_proj.weight")[kv]], dim=0)
        if qkv_bias:
            out[p + "bqkv"] = torch.cat([g(p + "q_proj.bias")[sl], g(p + "k_proj.bias")[kv], g(p + "v_proj.bias")[kv]], dim=0)
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


def _interleave64(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """Rows (or row scales) of the FP8 W13: 64-row blocks of gate and up alternating (the FP8 GEMM's tile is 128 wide)."""
    nb = gate.shape[0] // 64
    return torch.stack([gate.reshape(nb, 64, *gate.shape[1:]), up.reshape(nb, 64, *up.shape[1:])], dim=1).reshape(2 * nb * 64, *gate.shape[1:])


def shard_state_dict_fp8(sd: Dict[str, torch.Tensor], n_layers: int, n_heads: int, rank: int, tp: int, quantize, *,
                         n_kv_heads: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Rank `rank`'s FP8 shard of the four block linears of every layer. `quantize(w)` maps a full bf16 weight [N, K] to its
    e4m3 bytes (uint8 [N, K]) and row scales (fp32 [N]) with one scale per row over the full K (mmdp_quantize_fp8 with group =
    K, or oracle.fp8's restatement); every weight is quantised WHOLE and then sliced, so that each byte and scale a rank holds is
    bitwise a slice of the single-GPU FP8 context's weights:
      * column-parallel (q/k/v_proj as shard_state_dict's rows, ff_proj / up_proj): the rank's rows and their row scales; W13
        interleaves 64-row blocks of gate and up inside the shard (the FP8 GEMM's 128-wide SwiGLU tile);
      * row-parallel (attn_out, ff_out): the rank's K-columns of the bytes and the FULL row scales [d].
    Keys `blocks.i.` + wqkv8 / sqkv, wo8 / so, w13_8 / s13, w2_8 / s2."""
    g = lambda n: sd["model.transformer." + n] if ("model.transformer." + n) in sd else sd[n]
    da = (n_heads // tp) * 128
    kv0, n_kv_local = kv_shard(n_heads, n_kv_heads or n_heads, rank, tp)
    sl, kv = slice(rank * da, (rank + 1) * da), slice(kv0 * 128, (kv0 + n_kv_local) * 128)
    out = {}
    for i in range(n_layers):
        p = f"blocks.{i}."
        (qq, sq), (qk, sk), (qv, sv) = (quantize(g(p + n + ".weight")) for n in ("q_proj", "k_proj", "v_proj"))
        out[p + "wqkv8"] = torch.cat([qq[sl], qk[kv], qv[kv]]).contiguous()
        out[p + "sqkv"] = torch.cat([sq[sl], sk[kv], sv[kv]]).contiguous()
        qo, so = quantize(g(p + "attn_out.weight"))
        out[p + "wo8"], out[p + "so"] = qo[:, sl].contiguous(), so.contiguous()
        (q1, s1), (q3, s3) = quantize(g(p + "ff_proj.weight")), quantize(g(p + "up_proj.weight"))
        ff = q1.shape[0]
        if (ff // tp) % 128:
            raise ValueError("mlp_hidden / tp must be a multiple of 128 (SwiGLU tile interleave)")
        fs = slice(rank * (ff // tp), (rank + 1) * (ff // tp))
        out[p + "w13_8"] = _interleave64(q1[fs], q3[fs]).contiguous()
        out[p + "s13"] = _interleave64(s1[fs], s3[fs]).contiguous()
        q2, s2 = quantize(g(p + "ff_out.weight"))
        out[p + "w2_8"], out[p + "s2"] = q2[:, fs].contiguous(), s2.contiguous()
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
                 codebook_size: int = 8192, collective: str = "p2p", chunks: Optional[int] = None, precision: str = "bf16"):
        if precision not in ("bf16", "fp8"):
            raise ValueError(f"precision must be 'bf16' or 'fp8' (e4m3 block linears), not {precision!r}")
        self.precision = precision
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
        self.n_kv_heads = check_supported_config(config, self.n_heads, grouped_query=True)
        self.qkv_bias = bool(g("include_qkv_bias", False))
        self.h_local = self.n_heads // tp_size
        self.d_attn = self.h_local * 128
        if self.d_attn % 256:
            raise ValueError("n_heads / tp must be even (the fused QKV+RoPE epilogue works on 2-head tiles)")
        self.kv_local = kv_shard(self.n_heads, self.n_kv_heads, tp_rank, tp_size)[1]
        # a grouped-query or biased shard runs the grouped-query QKV epilogue and attention; the multi-head shard keeps its kernels
        self.gqa = self.kv_local != self.h_local or self.qkv_bias
        self.ff_local = self.ff // tp_size
        self.v_local = self.vocab_rows // tp_size
        self.vq_col0, self.vq_cols = text_vocab_size, codebook_size
        self.c_local = codebook_size // tp_size
        self.max_seq_len = int(max_seq_len or g("max_sequence_length", 4096))
        self.max_batch = max_batch
        sh = shard_state_dict(state_dict, self.n_layers, self.n_heads, tp_rank, tp_size, text_vocab_size, codebook_size,
                              n_kv_heads=self.n_kv_heads, qkv_bias=self.qkv_bias)
        fp8 = precision == "fp8"
        if fp8:  # the bf16 linears are not kept: their FP8 shards replace them
            sh = {k: v for k, v in sh.items() if k.split(".")[-1] not in ("wqkv", "wo", "w13", "w2")}
        self.w = {k: v.detach().to(device=self.device, dtype=torch.bfloat16).contiguous() for k, v in sh.items()}
        if fp8:
            self.w.update(shard_state_dict_fp8(state_dict, self.n_layers, self.n_heads, tp_rank, tp_size, self._quantize_rows,
                                               n_kv_heads=self.n_kv_heads))
        cos, sin = rope_tables(128, float(g("rope_theta", 10000.0)), self.max_seq_len)
        self.cos, self.sin = cos.to(self.device), sin.to(self.device)
        M, d, bf = self.max_batch * self.max_seq_len, self.d_model, dict(dtype=torch.bfloat16, device=self.device)
        self.Mmax = M
        self.q = torch.empty((M, self.d_attn), **bf)
        self.k = torch.empty((M, self.kv_local * 128), **bf)
        self.att = torch.empty((M, self.d_attn), **bf)
        self.h = torch.empty((M, self.ff_local), **bf)
        if fp8:
            # the e4m3 copy of the input of a linear quantised on this rank (att, h; the NCCL path also xn) and its scales
            ka = max(self.d_model, self.d_attn, self.ff_local)
            self.a8 = torch.empty(M * ka, dtype=torch.uint8, device=self.device)
            self.a8s = torch.empty(M * ka // 128, dtype=torch.float32, device=self.device)
        self.vt = None
        self._vt_key = None
        # packed forwards: the device row map of the packed rows, and their own V^T buffer [max_batch][kv_local][128][Lpad] (allocated
        # on the first packed forward) with the pad-rule bookkeeping of csrc/api.cu's vt_prepare: _pvt_Lpad = the column stride it was
        # last zeroed for, _pvt_len[s] = the columns of block s written since then
        self._row_map = torch.empty((M, 2), dtype=torch.int32, device=self.device)
        self._pvt = None
        self._pvt_Lpad, self._pvt_len = 0, [0] * self.max_batch
        if self.collective == "p2p":
            self._init_peer_buffers(group)
        else:
            self.x = torch.empty((M, d), **bf)
            self.xn = torch.empty((M, d), **bf)
            self.part = torch.empty((M, d), dtype=torch.float32, device=self.device)

    def _init_peer_buffers(self, group) -> None:
        """The peer-memory state of the "p2p" collective (csrc/tp_collective.cu): receive buffers, flags and the shared activation
        buffers of every row chunk, exported to and imported from the other ranks of `group`. Every rank calls it together."""
        M, d, tp_size, tp_rank = self.Mmax, self.d_model, self.tp, self.rank
        fp8 = self.precision == "fp8"
        bf = dict(dtype=torch.bfloat16, device=self.device)
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
        self._xq = None
        if fp8:
            # the e4m3 activation buffer every reduce but the last broadcasts into: [M, d] bytes, then M * d / 128 scales
            self._xq = _SharedBuffer(M * d + M * (d // 128) * 4, tp_rank, tp_size, group)
            self._xq_arr = (C.c_void_p * tp_size)(*self._xq.ptrs)
            self._xs_arr = (C.c_void_p * tp_size)(*[q + M * d for q in self._xq.ptrs])
        self.x = self._chunk_state[0]["x"]
        self._epoch = 0
        torch.cuda.synchronize()
        dist.barrier(group=group)  # every rank has mapped every buffer before the first peer access

    def __del__(self):
        shared = [getattr(self, "_xn", None), getattr(self, "_xq", None)]
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

    def _quantize_rows(self, w: torch.Tensor):
        """One full weight [N, K] -> (e4m3 bytes uint8 [N, K], row scales fp32 [N]) on this rank's device: mmdp_quantize_fp8 with
        one group per row, the quantisation of the single-GPU FP8 context's mmdp_model_set_weight."""
        q, s = _lib.quantize_fp8(w.detach().to(device=self.device, dtype=torch.bfloat16).contiguous(), group=w.shape[1])
        return q.view(torch.uint8), s[0]

    def _quantize_input(self, a: torch.Tensor, M: int, K: int, s):
        """The bf16 input [M, K] of an FP8 linear -> e4m3 bytes and 1 x 128 group scales in a8 / a8s."""
        check(lib.mmdp_quantize_fp8(ptr(a), K, M, K, 128, ptr(self.a8), K, ptr(self.a8s), s))

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
    def _packed_qkv_attention(self, p: str, packed, Lpad: int, a8=None, a8s=None):
        """QKV + RoPE and attention of layer prefix `p` over the packed batch packed = (n_seg, host int32 lengths) on the NCCL path:
        mmdp_qkv_rope_tp_packed on xn (bf16) or on its e4m3 copy a8 / a8s (FP8), then the packed attention."""
        d, s, w = self.d_model, stream_ptr(), self.w
        n, lens = packed
        if a8 is None:
            prec, a, sa, wq, sw = _lib.PRECISION_BF16, ptr(self.xn), None, ptr(w[p + "wqkv"]), None
        else:
            prec, a, sa, wq, sw = _lib.PRECISION_FP8, a8, a8s, ptr(w[p + "wqkv8"]), ptr(w[p + "sqkv"])
        check(lib.mmdp_qkv_rope_tp_packed(prec, a, d, sa, wq, sw, ptr(w.get(p + "bqkv")), d, self.h_local, self.kv_local, n, lens, Lpad,
                                          ptr(self.cos), ptr(self.sin), ptr(self.q), ptr(self.k), ptr(self._pvt), ptr(self._row_map), s))
        check(lib.mmdp_attention_gqa(ptr(self.q), ptr(self.k), ptr(self._pvt), ptr(self.att), n, lens, self.h_local, self.kv_local, 0,
                                     Lpad, 1.0 / math.sqrt(128.0), s))

    def _layers_nccl(self, B: int, L: int, M: int, Lpad: int, packed=None):
        """Round 1's formulation, kept as the measured baseline (`collective="nccl"`): fp32 partial sums stored locally,
        `dist.all_reduce` between the kernels, then the residual add and the RMSNorm as separate launches. packed: (n_seg, host
        int32 lengths) of a packed batch of M rows (B, L unused), or None."""
        d, s, w = self.d_model, stream_ptr(), self.w
        scale = 1.0 / math.sqrt(128.0)
        x, xn = self.x, self.xn
        if self.precision == "fp8":
            return self._layers_nccl_fp8(B, L, M, Lpad, packed)
        for i in range(self.n_layers):
            p = f"blocks.{i}."
            check(lib.mmdp_rmsnorm(ptr(x), d, None, ptr(w[p + "attn_norm"]), ptr(xn), d, M, d, self.rms_eps, s))
            if packed is not None:
                self._packed_qkv_attention(p, packed, Lpad)
            elif self.gqa:
                check(lib.mmdp_qkv_rope_tp_gqa(ptr(xn), d, ptr(w[p + "wqkv"]), ptr(w.get(p + "bqkv")), M, d, self.h_local, self.kv_local,
                                               L, Lpad, ptr(self.cos), ptr(self.sin), ptr(self.q), ptr(self.k), ptr(self.vt), s))
                check(lib.mmdp_attention_gqa(ptr(self.q), ptr(self.k), ptr(self.vt), ptr(self.att), B, None, self.h_local, self.kv_local,
                                             L, Lpad, scale, s))
            else:
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

    def _layers_nccl_fp8(self, B: int, L: int, M: int, Lpad: int, packed=None):
        """_layers_nccl with the four linears in FP8: each bf16 input is quantised (1 x 128 groups) right before its GEMM."""
        d, s, w, da, ffl = self.d_model, stream_ptr(), self.w, self.d_attn, self.ff_local
        scale = 1.0 / math.sqrt(128.0)
        x, xn, a8, a8s = self.x, self.xn, ptr(self.a8), ptr(self.a8s)
        for i in range(self.n_layers):
            p = f"blocks.{i}."
            check(lib.mmdp_rmsnorm(ptr(x), d, None, ptr(w[p + "attn_norm"]), ptr(xn), d, M, d, self.rms_eps, s))
            self._quantize_input(xn, M, d, s)
            if packed is not None:
                self._packed_qkv_attention(p, packed, Lpad, a8, a8s)
            else:
                check(lib.mmdp_qkv_rope_tp_fp8(a8, d, a8s, ptr(w[p + "wqkv8"]), ptr(w[p + "sqkv"]), ptr(w.get(p + "bqkv")), M, d, self.h_local,
                                               self.kv_local, L, Lpad, ptr(self.cos), ptr(self.sin), ptr(self.q), ptr(self.k), ptr(self.vt), s))
                if self.gqa:
                    check(lib.mmdp_attention_gqa(ptr(self.q), ptr(self.k), ptr(self.vt), ptr(self.att), B, None, self.h_local, self.kv_local,
                                                 L, Lpad, scale, s))
                else:
                    check(lib.mmdp_attention(ptr(self.q), ptr(self.k), ptr(self.vt), ptr(self.att), B, self.h_local, L, Lpad, scale, s))
            self._quantize_input(self.att, M, da, s)
            check(lib.mmdp_gemm_fp8_f32(a8, da, a8s, ptr(w[p + "wo8"]), da, ptr(w[p + "so"]), M, d, da, ptr(self.part), d, s))
            self._allreduce(self.part[:M])
            check(lib.mmdp_resid_add_f32(ptr(x), d, ptr(self.part), d, M, d, s))
            check(lib.mmdp_rmsnorm(ptr(x), d, None, ptr(w[p + "ff_norm"]), ptr(xn), d, M, d, self.rms_eps, s))
            self._quantize_input(xn, M, d, s)
            check(lib.mmdp_gemm_fp8(EPI_SWIGLU, a8, d, a8s, ptr(w[p + "w13_8"]), d, ptr(w[p + "s13"]), M, 2 * ffl, d, ptr(self.h), ffl,
                                    None, 0, s))
            self._quantize_input(self.h, M, ffl, s)
            check(lib.mmdp_gemm_fp8_f32(a8, ffl, a8s, ptr(w[p + "w2_8"]), ffl, ptr(w[p + "s2"]), M, d, ffl, ptr(self.part), d, s))
            self._allreduce(self.part[:M])
            check(lib.mmdp_resid_add_f32(ptr(x), d, ptr(self.part), d, M, d, s))

    def _native_ctx(self, B: int, L: int):
        """The C-side description of this rank (mmdp_tp_ctx): built once per (B, L) - the V^T buffer depends on it."""
        key = (B, L)
        if getattr(self, "_ctx_key", None) == key:
            return self._ctx
        split = chunk_split(B * L) if self.chunks == 2 else [B * L]
        self._ctx, self._ctx_layers = self._make_ctx(self.vt, split)
        self._ctx_key = key
        return self._ctx

    def _make_ctx(self, vt: torch.Tensor, split: List[int]):
        """mmdp_tp_ctx of this rank over the V^T buffer `vt` and the row chunks `split`; returns it with the layer arrays it points
        to (the caller keeps them alive)."""
        w = self.w
        layers = (_lib.TpLayer * self.n_layers)()
        fp8 = self.precision == "fp8"
        layers8 = (_lib.TpLayerFp8 * self.n_layers)() if fp8 else None
        for i in range(self.n_layers):
            p = f"blocks.{i}."
            names = ("attn_norm", "ff_norm") if fp8 else ("wqkv", "wo", "w13", "w2", "attn_norm", "ff_norm")
            for name in names:
                setattr(layers[i], name, w[p + name].data_ptr())
            if fp8:
                for name, key in (("wqkv", "wqkv8"), ("wo", "wo8"), ("w13", "w13_8"), ("w2", "w2_8"), ("sqkv", "sqkv"), ("so", "so"),
                                  ("s13", "s13"), ("s2", "s2")):
                    setattr(layers8[i], name, w[p + key].data_ptr())
            if self.qkv_bias:
                layers[i].bqkv = w[p + "bqkv"].data_ptr()
        c = _lib.TpCtx()
        c.d_model, c.n_heads_local, c.ff_local, c.n_layers, c.n_ranks, c.rank = self.d_model, self.h_local, self.ff_local, self.n_layers, self.tp, self.rank
        c.n_kv_heads_local = self.kv_local
        c.rms_eps = self.rms_eps
        c.layers = layers
        c.wte, c.ln_f, c.vocab = w["wte"].data_ptr(), w["ln_f"].data_ptr(), w["wte"].shape[0]
        c.cos_tab, c.sin_tab = self.cos.data_ptr(), self.sin.data_ptr()
        c.q, c.k, c.att, c.h, c.vt = self.q.data_ptr(), self.k.data_ptr(), self.att.data_ptr(), self.h.data_ptr(), vt.data_ptr()
        c.xn = C.cast(self._xn.array, C.POINTER(C.c_void_p))
        if fp8:
            c.precision = _lib.PRECISION_FP8
            c.layers_fp8 = layers8
            c.xq = C.cast(self._xq_arr, C.POINTER(C.c_void_p))
            c.xq_scales = C.cast(self._xs_arr, C.POINTER(C.c_void_p))
            c.a8, c.a8_scales = self.a8.data_ptr(), self.a8s.data_ptr()
        c.n_chunks = len(split)
        c.chunk_rows0 = split[0]
        c.packed.seg_pos, c.packed.max_rows, c.packed.rope_len = self._row_map.data_ptr(), self.Mmax, self.max_seq_len
        for ci in range(self._alloc_chunks):  # both chunks' buffers: a packed forward picks its split per call
            st = self._chunk_state[ci]
            c.chunk[ci].x_shard = st["x"].data_ptr()
            c.chunk[ci].recv[0] = C.cast(st["recv"][0].array, C.POINTER(C.c_void_p))
            c.chunk[ci].recv[1] = C.cast(st["recv"][1].array, C.POINTER(C.c_void_p))
            c.chunk[ci].flags = C.cast(st["flags"].array, C.POINTER(C.c_void_p))
            c.chunk[ci].done_counter = st["done"].data_ptr()
        return c, (layers, layers8)

    def _final_norm(self, ids: torch.Tensor) -> torch.Tensor:
        """Runs embedding + all blocks; returns ln_f(x) for ALL rows [M, d] (p2p) or the raw residual stream x (nccl)."""
        B, L = ids.shape
        M, d, s = B * L, self.d_model, stream_ptr()
        if M > self.Mmax:
            raise _lib.MmdpError("TensorParallelLLaDA: batch x length exceeds the workspace")
        Lpad = (L + 7) // 8 * 8
        if self._vt_key != (B, Lpad, L):
            self.vt = torch.zeros((B, self.kv_local, 128, Lpad), dtype=torch.bfloat16, device=self.device)
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

    def _prepare_packed_vt(self, lens: List[int], Lpad: int) -> None:
        """V^T pad rule of the packed buffer (csrc/api.cu, vt_prepare): block s is read up to Lpad and its columns [L_s, Lpad) must
        be zeros. The buffer is zeroed when the column stride changes or when one of the blocks held more columns than its new
        length; otherwise every column read past L_s is still zero. Packed and equal-length forwards alternate freely: the
        equal-length forward keeps its own buffer."""
        if self._pvt is None:
            rows = self.max_batch * self.kv_local * 128 * ((self.max_seq_len + 7) // 8 * 8)
            self._pvt = torch.zeros(rows, dtype=torch.bfloat16, device=self.device)
            if self.collective == "p2p":
                self._pctx = self._make_ctx(self._pvt, [1])   # built once; the row chunks are set per call
        if self._pvt_Lpad != Lpad or any(old > new for old, new in zip(self._pvt_len, lens)):
            self._pvt.zero_()
            self._pvt_len = [0] * self.max_batch
            self._pvt_Lpad = Lpad
        self._pvt_len[:len(lens)] = lens

    def _final_norm_packed(self, ids: torch.Tensor, lens: List[int]) -> torch.Tensor:
        """_final_norm over a packed batch (lengths already checked): ln_f(x) of all packed rows (p2p) or the raw x (nccl)."""
        M, d, s = sum(lens), self.d_model, stream_ptr()
        split = chunk_split(M) if (self.collective == "p2p" and self.chunks == 2) else [M]
        if self.collective == "p2p":
            for rows in split:
                if row_partition(rows, self.tp, self.tp - 1)[1] < 1:
                    raise ValueError(f"TensorParallelLLaDA: {rows} packed rows cannot be split over {self.tp} ranks with at least one row each")
        Lpad = (max(lens) + 7) // 8 * 8
        self._prepare_packed_vt(lens, Lpad)
        c_lens = (C.c_int32 * len(lens))(*lens)
        if self.collective == "p2p":
            c = self._pctx[0]
            c.n_chunks, c.chunk_rows0 = len(split), split[0]
            out = C.c_uint32(0)
            check(lib.mmdp_tp_forward_packed(C.byref(c), ptr(ids), len(lens), c_lens, self._epoch, C.byref(out), s))
            self._epoch = int(out.value)
            return self.xn
        wte = self.w["wte"]
        check(lib.mmdp_embed(ptr(ids), ptr(wte), ptr(self.x), M, d, wte.shape[0], s))
        self._layers_nccl(0, 0, M, Lpad, packed=(len(lens), c_lens))
        return self.x

    @torch.no_grad()
    def forward_rows(self, ids: torch.Tensor, rows_a: Optional[torch.Tensor] = None, rows_b: Optional[torch.Tensor] = None,
                     col0_b: int = 0, ncols_b: int = 0, out_a: Optional[torch.Tensor] = None, out_b: Optional[torch.Tensor] = None):
        hid = self._final_norm(ids.contiguous())
        return self._head(hid, rows_a, rows_b, col0_b, ncols_b, out_a, out_b)

    @torch.no_grad()
    def forward_rows_packed(self, ids_packed: torch.Tensor, seq_lens, rows_a: Optional[torch.Tensor] = None,
                            rows_b: Optional[torch.Tensor] = None, col0_b: int = 0, ncols_b: int = 0,
                            out_a: Optional[torch.Tensor] = None, out_b: Optional[torch.Tensor] = None, row_windows=None):
        """One forward over a packed batch: ids_packed [sum(seq_lens)] holds the sequences end to end, each computed as if it were
        alone (attention stays inside it, positions restart at 0), the contract of LLaDAForMultiModalGeneration.forward_rows_packed.
        rows_* are int32 packed row indices; the LM head is forward_rows'. At most max_batch sequences (and 64), each at most
        max_seq_len long: ValueError before anything is launched. The tensor-parallel model has no row windows (row_windows must
        be None)."""
        if row_windows is not None:
            raise NotImplementedError("the tensor-parallel model has no last-block row windows")
        lens = [int(x) for x in seq_lens]
        if not lens or len(lens) > min(self.max_batch, 64):
            raise ValueError(f"a packed forward takes 1 to max_batch={self.max_batch} (at most 64) sequences, got {len(lens)}")
        if min(lens) < 1 or max(lens) > self.max_seq_len:
            raise ValueError(f"packed sequence lengths must lie in [1, max_seq_len={self.max_seq_len}], got {lens}")
        if ids_packed.numel() != sum(lens):
            raise ValueError(f"ids_packed holds {ids_packed.numel()} tokens, the sequence lengths add up to {sum(lens)}")
        hid = self._final_norm_packed(ids_packed.to(device=self.device, dtype=torch.int64).contiguous(), lens)
        return self._head(hid, rows_a, rows_b, col0_b, ncols_b, out_a, out_b)

    def _head(self, hid: torch.Tensor, rows_a, rows_b, col0_b: int, ncols_b: int, out_a, out_b):
        """The LM head on the rows of `hid` (_final_norm's result): vocabulary slices of this rank, all-gathered."""
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
