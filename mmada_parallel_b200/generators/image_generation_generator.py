"""Drop-in for MMaDA-Parallel-A/generators/image_generation_generator.py: `generate_image`, MaskGit parallel decoding of the VQ
tokens of a text-to-image prompt (SURVEY.md section 8f rank 3). Same name, keyword-only arguments, defaults and return value
(`LongTensor [1, seq_len]` of FULL-vocabulary ids, newlines removed) as the reference function (:15-251).

Per step (reference lines in brackets) the host does: count / locate the masked positions (one device->host read, where the
reference has several `.item()`s) [:92], evaluate the keep-count from the schedule on the CPU [:99-103], run the conditional and
(cfg_scale > 0) unconditional forwards with the LM head restricted to the masked rows x the codebook window [:121-162], draw
the two uniform noise tensors from the caller's generator with the reference's calls [generation_utils.py:28-34], and launch
`mmdp_image_step_t2i` (CFG mix, Gumbel-max sample, softmax confidence, write-back, re-mask) [:171-208].

`use_cache=True` is accepted: the reference enables its per-block K/V and logit caches [:65-68] but never hands
`to_compute_mask` / `cat` to the model (the wrapper's forward has no such parameter, modeling_xllmx_dimoo.py:41-72; the masks
computed at :224-239 are dead values), so every forward recomputes all tokens and the cache stores are invisible: outputs with
and without the flag are identical in the reference, and here.
"""
from __future__ import annotations

import os
from typing import Callable, Optional

import torch

from .._lib import check, lib, ptr, stream_ptr
from ..schedule import cosine_schedule
from .parallel_generator import MAX_CODEBOOK, MAX_VQ_TOKENS

__all__ = ["generate_image", "cosine_schedule"]


@torch.no_grad()
def generate_image(
    model,
    prompt: torch.LongTensor,
    *,
    seq_len: int = 1024,
    newline_every: int = 16,
    timesteps: int = 18,
    mask_token_id: int = 126336,
    newline_id: int = 126084,
    temperature: float = 1.0,
    cfg_scale: float = 0.0,
    uncon_ids: torch.LongTensor = None,
    code_start: Optional[int] = None,
    codebook_size: int = 8192,
    noise_schedule: Callable[[torch.Tensor], torch.Tensor] = cosine_schedule,
    text_vocab_size: Optional[int] = None,
    generator: Optional[torch.Generator] = None,
    use_cache=False,
    cache_ratio=0.9,
    refresh_interval=5,
    warmup_ratio=0.3,
    debug: bool = True,
    debug_log_dir: Optional[str] = None,
    max_print_tokens: int = 100,
    _trace: Optional[list] = None,
) -> torch.LongTensor:
    if not hasattr(model, "forward_rows"):
        raise TypeError("generate_image needs a mmada_parallel_b200.model.LLaDAForMultiModalGeneration (H100-native) model")
    if debug and debug_log_dir:
        os.makedirs(debug_log_dir, exist_ok=True)
    device = model.device
    prompt = prompt.to(device=device, dtype=torch.int64)
    B, P = prompt.shape
    assert B == 1, "batch>1 not supported – wrap in loop if needed"                              # :57
    if codebook_size > MAX_CODEBOOK or codebook_size % 8:
        raise ValueError(f"codebook_size must be a multiple of 8 and <= {MAX_CODEBOOK} (got {codebook_size})")
    x = prompt.clone().contiguous()
    if hasattr(model, "caching"):
        model.caching(use_cache)                                                                 # :65-68
    if text_vocab_size is None:                                                                  # :78-82
        text_vocab_size = model.vocab_rows - codebook_size
    off = int(text_vocab_size)
    vq_len = int((x == mask_token_id).sum())                                                     # :61-63 (one read-back)
    if vq_len > MAX_VQ_TOKENS:
        raise ValueError(f"at most {MAX_VQ_TOKENS} masked VQ positions are supported (got {vq_len})")
    use_cfg = cfg_scale > 0
    if use_cfg:
        if uncon_ids is None or code_start is None:
            raise ValueError("cfg_scale > 0 needs uncon_ids and code_start")
        unc_prefix = uncon_ids.to(device=device, dtype=torch.int64)
        shift = unc_prefix.shape[1] - (code_start - 2)
        uncond = torch.empty((1, unc_prefix.shape[1] + P - (code_start - 2)), dtype=torch.int64, device=device)
        uncond[:, : unc_prefix.shape[1]] = unc_prefix
    gdev = generator.device if generator is not None else device
    cap = max(vq_len, 1)
    cond_vq = torch.empty((cap, codebook_size), dtype=torch.bfloat16, device=device)
    unc_vq = torch.empty_like(cond_vq) if use_cfg else None
    sampled_ws = torch.empty(cap, dtype=torch.int32, device=device)
    selp_ws = torch.empty(cap, dtype=torch.float32, device=device)
    unk_ws = torch.empty(cap, dtype=torch.uint8, device=device)
    if debug:   # (the reference prints shapes and token samples per step; this mirror reports the per-step counts only)
        print(f"[generate_image] {device}: {vq_len} masked VQ positions of {seq_len}, {timesteps} steps, vocab offset {off}, "
              f"codebook {codebook_size}, cfg {cfg_scale}")
    for step in range(timesteps):
        flat_idx = (x[0] == mask_token_id).nonzero(as_tuple=False)[:, 0]                         # the step's read-back (:92)
        n = int(flat_idx.numel())
        if n == 0:                                                                               # :92-95 early exit
            if debug:
                print(f"[generate_image] step {step}: nothing left to fill")
            break
        if step < timesteps - 1:                                                                 # :99-103, on the CPU like the oracle
            frac = noise_schedule(torch.tensor([(step + 1) / timesteps]))
            keep_n = int((torch.tensor([[float(vq_len)]]) * frac).floor().clamp_min(1).long())
        else:
            keep_n = 0
        if debug:
            print(f"[generate_image] step {step}: {n} masked, {keep_n} stay masked")
        rows = flat_idx.to(torch.int32)
        model.forward_rows(x, rows_b=rows, col0_b=off, ncols_b=codebook_size, out_b=cond_vq[:n])  # :127 / :158
        if use_cfg:
            if int(flat_idx[0]) < code_start - 2:
                raise ValueError("masked positions before code_start - 2 cannot be aligned with the unconditional sequence")
            uncond[:, unc_prefix.shape[1]:] = x[:, code_start - 2:]                              # :123
            model.forward_rows(uncond, rows_b=(rows + shift), col0_b=off, ncols_b=codebook_size, out_b=unc_vq[:n])   # :141
        # gumbel_noise(): torch.rand(t.shape, dtype=t.dtype, generator=generator) - logits [1, n, C] first (only when tau != 0),
        # then the confidences [1, n] (always)                                                   (generation_utils.py:28-42, :52)
        u1 = None
        if temperature != 0.0:
            u1 = torch.rand((1, n, codebook_size), dtype=torch.bfloat16, device=gdev, generator=generator).to(device)
        u2 = torch.rand((1, n), dtype=torch.bfloat16, device=gdev, generator=generator).to(device)
        check(lib.mmdp_image_step_t2i(ptr(cond_vq), ptr(unc_vq), codebook_size, n, codebook_size, float(cfg_scale), ptr(u1),
                                      float(temperature), ptr(u2), float(temperature), keep_n, ptr(x), ptr(rows), int(mask_token_id),
                                      off, ptr(sampled_ws), ptr(selp_ws), ptr(unk_ws), None, stream_ptr()))
        if _trace is not None:
            # (the reference clamps keep_n to n - 1 IN PLACE inside mask_by_random_topk, generation_utils.py:57; the kernel clamps too)
            _trace.append(dict(step=step, keep_n=min(keep_n, n - 1), sampled=sampled_ws[:n].long().clone(), x=x[0].clone()))
        if debug and debug_log_dir:
            import numpy as np
            base = os.path.join(debug_log_dir, f"step_{step}")
            np.save(base + "_x.npy", x.cpu().numpy())
            np.save(base + "_vq_mask.npy", (x == mask_token_id).cpu().numpy())
            np.save(base + "_sampled_full.npy", (sampled_ws[:n].long() + off).cpu().numpy())
    if hasattr(model, "raise_device_errors"):
        model.raise_device_errors()
    vq_ids = x[0, code_start:-2]                                                                 # :236-238
    vq_ids = vq_ids[vq_ids != newline_id].view(1, seq_len)
    if debug:
        print(f"[generate_image] done: ids {tuple(vq_ids.shape)}")
    return vq_ids
