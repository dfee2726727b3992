"""ORACLE (test infrastructure, NOT product code): CPU restatement of the reference's mask-predict step.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this package.
Every function restates reference code (file:line given) with torch-CPU ops so that dtypes, rounding points and
tie rules are the reference's own. Random numbers are explicit inputs: `NoiseSource` draws them from a
torch.Generator with exactly the calls (shape, dtype, order) the reference makes, so a replayed generator reproduces
the reference trajectory. Pinned against the real reference by oracle/make_golden.py -> tests/golden/*.pt
(tests/test_oracle_golden.py).
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

MASK_TOKEN_A = 126336
NEW_LINE_A = 126084


# ---------------------------------------------------------------------------------------------------------------
# schedules / host-side integer helpers
# ---------------------------------------------------------------------------------------------------------------
def cosine_schedule(t: torch.Tensor) -> torch.Tensor:
    """A/generators/parallel_generator.py:73-75 == M/models/sampling.py:39-40."""
    return torch.cos(t * math.pi / 2)


def get_num_transfer_tokens_a(n_masked: int, text_steps: int) -> list:
    """A/generators/parallel_generator.py:78-99 (floor-based), one batch row."""
    out, remaining = [], n_masked
    for step in range(text_steps):
        ratio = (step + 1) / text_steps
        target_remaining = int(n_masked * (1 - ratio))
        k = max(0, remaining - target_remaining)
        out.append(k)
        remaining -= k
    return out


def get_num_transfer_tokens_m(n_masked: int, steps: int) -> list:
    """M/models/modeling_mmada.py:63-81 (base + remainder)."""
    base, rem = n_masked // steps, n_masked % steps
    return [base + (1 if i < rem else 0) for i in range(steps)]


def image_step_indices(text_steps: int, timesteps: int) -> list:
    """A/generators/parallel_generator.py:157-159 == M/models/modeling_mmada.py:161."""
    return torch.linspace(text_steps // 4, text_steps - 1, timesteps).round().int().tolist()


def sched_len(num_vq_tokens: int, step: int, text_steps: int, noise_schedule=cosine_schedule) -> int:
    """floor(N * noise_schedule(ratio)) on a 0-d fp32 tensor (parallel_generator.py:318-322; modeling_mmada.py:226-233).
    At ratio == 1 the fp32 cosine is -4.37e-8 -> floor gives -1 (then clamped to 1 by the caller)."""
    ratio = 1.0 * (step + 1) / text_steps
    mask_ratio = noise_schedule(torch.tensor(ratio))
    return int((num_vq_tokens * mask_ratio).floor().item())


# ---------------------------------------------------------------------------------------------------------------
# noise, drawn exactly like the reference draws it
# ---------------------------------------------------------------------------------------------------------------
class NoiseSource:
    """Replays the reference's RNG calls on `generator` (CPU or CUDA). All tensors are created on generator.device."""

    def __init__(self, generator: Optional[torch.Generator], dtype=torch.bfloat16):
        self.g = generator
        self.dtype = dtype
        self.device = generator.device if generator is not None else torch.device("cpu")

    def text_uniform(self, shape):
        """torch.rand(logits.shape, dtype=logits.dtype, generator=...)  (parallel_generator.py:13-14)"""
        return torch.rand(shape, dtype=self.dtype, device=self.device, generator=self.g)

    def multinomial_q(self, n_rows: int, n_cols: int):
        """The `q` of torch.multinomial(probs, 1, generator) (parallel_generator.py:299-300; modeling_mmada.py:222):
        ATen draws q = empty_like(probs).exponential_(1, gen) and returns argmax(probs / q)."""
        return torch.empty((n_rows, n_cols), dtype=self.dtype, device=self.device).exponential_(1, generator=self.g)

    def remask_randn(self, shape):
        """torch.randn(probs.shape, dtype=probs.dtype, generator=...)  (parallel_generator.py:30-31)"""
        return torch.randn(shape, dtype=self.dtype, device=self.device, generator=self.g)

    def remask_uniform(self, shape):
        """torch.zeros_like(t).uniform_(0, 1, generator=generator)  (M/models/sampling.py:14-15)"""
        return torch.zeros(shape, dtype=self.dtype, device=self.device).uniform_(0, 1, generator=self.g)


# ---------------------------------------------------------------------------------------------------------------
# text step
# ---------------------------------------------------------------------------------------------------------------
def add_gumbel_noise_a(logits: torch.Tensor, temperature: float, uniform_noise: Optional[torch.Tensor]):
    """A/generators/parallel_generator.py:8-20 with the uniform draw made explicit."""
    if temperature == 0:
        return logits
    gumbel_noise = -torch.log(-torch.log(uniform_noise + 1e-10) + 1e-10)
    return logits + temperature * gumbel_noise


def add_gumbel_noise_m(logits: torch.Tensor, temperature: float, uniform64: Optional[torch.Tensor] = None):
    """M/models/modeling_mmada.py:49-60: fp64 Gumbel-max, exp(logits) / (-log u)^temperature with u = torch.rand_like(logits,
    dtype=float64) drawn from the GLOBAL RNG of the logits' device (explicit here when `uniform64` is given)."""
    if temperature == 0:
        return logits
    logits = logits.to(torch.float64)
    noise = torch.rand_like(logits, dtype=torch.float64) if uniform64 is None else uniform64
    gumbel_noise = (-torch.log(noise)) ** temperature
    return logits.exp() / gumbel_noise


def text_step(text_logits: torch.Tensor, ids_text: torch.Tensor, mask_id: int, k: int,
              uncond_logits: Optional[torch.Tensor] = None, text_cfg: float = 0.0, temperature: float = 0.0,
              uniform_noise: Optional[torch.Tensor] = None, uniform64: Optional[torch.Tensor] = None, gumbel_m: bool = False):
    """One text un-masking step for one batch row.
    A: parallel_generator.py:181-217 (logits = cond).  M: modeling_mmada.py:179-209 (logits = cond + cfg*(uncond-cond)).
    text_logits [R, V] (bf16), ids_text [R] int64 (modified copy returned). Returns (new_ids, x0, confidence)."""
    logits = text_logits
    if uncond_logits is not None:
        logits = text_logits + text_cfg * (uncond_logits - text_logits)          # modeling_mmada.py:179
    masked = ids_text == mask_id
    if gumbel_m or uniform64 is not None:
        logits_with_noise = add_gumbel_noise_m(logits, temperature, uniform64)       # modeling_mmada.py:185 / :659
    else:
        logits_with_noise = add_gumbel_noise_a(logits, temperature, uniform_noise)
    x0 = torch.argmax(logits_with_noise, dim=-1)                                  # :189
    p = F.softmax(logits.to(torch.float64), dim=-1)                              # :193
    x0_p = torch.squeeze(torch.gather(p, dim=-1, index=torch.unsqueeze(x0, -1)), -1)
    x0 = torch.where(masked, x0, ids_text)                                        # :204
    confidence = torch.where(masked, x0_p, -np.inf)                               # :205
    new_ids = ids_text.clone()
    if k > 0:
        # torch.topk's order among equal confidences is unspecified; the product uses "larger value, then lower
        # index". Ties only occur between -inf entries (un-masked positions, whose x0 is the id already there).
        order = sorted(range(confidence.numel()), key=lambda i: (-float(confidence[i]), i))
        sel = torch.tensor(order[:k], dtype=torch.long)
        new_ids[sel] = x0[sel]                                                    # :212-217
    return new_ids, x0, x0_p


# ---------------------------------------------------------------------------------------------------------------
# image step
# ---------------------------------------------------------------------------------------------------------------
def image_logits_a(cond, unc_text, unc_img, cfg_scale: float, cfg_img: float):
    """parallel_generator.py:282-289."""
    image_logits = cond
    if not (cfg_scale == 0.0 and cfg_img == 0.0):
        if cfg_scale != 0.0:
            image_logits = image_logits + cfg_scale * (cond - unc_text)
        if cfg_img != 0.0:
            image_logits = image_logits + cfg_img * (cond - unc_img)
    return image_logits


def image_logits_m(cond, uncond, image_cfg: float):
    """modeling_mmada.py:216."""
    return (1 + image_cfg) * cond - image_cfg * uncond


def sample_rows(probs: torch.Tensor, q: Optional[torch.Tensor]):
    """argmax(probs) at temperature 0 (parallel_generator.py:294-295) or torch.multinomial(probs, 1) restated with its
    exponential draw q made explicit (ATen multinomial fast path: argmax(probs / q))."""
    if q is None:
        return probs.argmax(dim=-1)
    return (probs / q).argmax(dim=-1)


def mask_by_random_topk_a(mask_len: int, probs: torch.Tensor, temperature: float, noise: Optional[torch.Tensor],
                          stable: bool = False):
    """parallel_generator.py:23-70 for batch 1 with the randn draw explicit. probs [N] -> bool [N].
    stable=False issues the reference's own call, torch.sort(confidence, descending=False): its order among EQUAL
    bf16 confidences is implementation-defined (on an AVX-512 CPU ATen uses an unstable SIMD sort; the CUDA backend
    orders differently again), so which of several tied tokens stays masked is not a property of the algorithm.
    stable=True is the deterministic rule the H100 kernel implements (ties -> lower index first)."""
    if noise is None:
        noise = torch.zeros_like(probs)
    confidence = torch.log(probs + 1e-10) + temperature * noise
    _, sorted_indices = torch.sort(confidence.unsqueeze(0), dim=-1, descending=False, stable=stable)
    sorted_indices = sorted_indices[0]
    k = int(min(max(mask_len, 0), probs.shape[-1] - 1))                            # :43
    masking = torch.zeros_like(probs, dtype=torch.bool)
    if k > 0:
        masking[sorted_indices[:k]] = True
    return masking, confidence


def _log_m(t, eps=1e-20):
    return torch.log(t.clamp(min=eps))                                            # M/models/sampling.py:10-11


def mask_by_random_topk_m(mask_len: int, probs: torch.Tensor, temperature: float, uniform: Optional[torch.Tensor]):
    """M/models/sampling.py:31-36 for batch 1 with the uniform draw explicit."""
    g = -_log_m(-_log_m(uniform)) if uniform is not None else torch.zeros_like(probs)
    confidence = _log_m(probs) + temperature * g
    sorted_confidence = torch.sort(confidence, dim=-1).values
    cut_off = sorted_confidence[int(mask_len)]
    return confidence < cut_off, confidence


def image_step(variant: str, cond: torch.Tensor, unc_a: Optional[torch.Tensor], unc_b: Optional[torch.Tensor],
               s_a: float, s_b: float, vq_state: torch.Tensor, mask_id: int, sched: int, temp: float,
               q: Optional[torch.Tensor], conf_noise: Optional[torch.Tensor], codebook_size: int, stable: bool = False):
    """One image step for one sample.
    variant "A": parallel_generator.py:220-344; cond/unc_a/unc_b = cond/uncond_text/uncond_image VQ logits [N, C],
                 s_a = cfg_scale, s_b = cfg_img. vq_state [N] int64: VQ id (already offset-removed & clamped) or -1 for masked.
    variant "M": modeling_mmada.py:211-241; unc_a = uncond logits, s_a = image_cfg; vq_state uses mask_id for masked.
    Returns dict(sampled, probs, selected_probs, mask_len, masking, final) - final[i] = -1 (stay masked) or VQ id."""
    N = cond.shape[0]
    if variant == "A":
        logits = image_logits_a(cond, unc_a, unc_b, s_a, s_b)
        unknown = vq_state == -1
    else:
        logits = image_logits_m(cond, unc_a, s_a)
        unknown = vq_state == mask_id
    probs = F.softmax(logits, dim=-1)                                              # :292 / M :219
    sampled = sample_rows(probs, q)
    sampled = torch.where(unknown, sampled, vq_state)                              # :305 / M :225
    if variant == "A":
        sampled = torch.clamp(sampled, 0, codebook_size - 1)                       # :308
    selected = torch.gather(probs, -1, sampled.long()[..., None]).squeeze(-1)      # :311
    high_val = torch.finfo(selected.dtype).max
    selected = torch.where(unknown, selected, high_val)                            # :314-315
    unknown_count = int(unknown.sum())
    mask_len = max(1, min(unknown_count - 1, sched))                               # :324 / M :234
    if variant == "A":
        masking, conf = mask_by_random_topk_a(mask_len, selected, temp, conf_noise, stable=stable)
    else:
        masking, conf = mask_by_random_topk_m(mask_len, selected, temp, conf_noise)
    final = torch.where(masking, torch.tensor(-1), sampled)
    return dict(sampled=sampled, probs=probs, selected_probs=selected, mask_len=mask_len, masking=masking,
                final=final, confidence=conf, unknown=unknown)


# ---------------------------------------------------------------------------------------------------------------
# VQ codebooks
# ---------------------------------------------------------------------------------------------------------------
def lfq_codebook_entry(indices: torch.Tensor, bits: int = 13) -> torch.Tensor:
    """LFQuantizer.get_codebook_entry (M/models/modeling_magvitv2.py:186-221): ids [B, N] -> [B, bits, h*w] (+-1.0)."""
    binary = (indices.unsqueeze(-1) >> torch.arange(bits - 1, -1, -1, dtype=torch.long)) & 1
    return (binary.float() * 2 - 1).permute(0, 2, 1).contiguous()
