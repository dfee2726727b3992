"""Drop-in for MMaDA-Parallel-A/generators/parallel_generator.py: same function names, signatures and return values.

`generate_ti2ti` keeps the reference's control flow (:102-368) but every per-step computation is a CUDA kernel of
libmmdp.so and the id sequence never leaves the GPU inside the loop:
  forward (restricted LM head)      -> mmdp_model_forward   (text rows x V, image rows x codebook columns only)
  text step   (:181-217)            -> mmdp_text_step       (argmax, fp64 softmax confidence, top-k commit)
  image step  (:220-344)            -> mmdp_image_step      (CFG mix, softmax, sample, confidence, re-mask, write-back)
The ~3 300 host<->device syncs per image step of the reference (.item() loops) are gone: the only host work per step
is launching kernels and, when sampling is stochastic, drawing the noise tensors from the caller's torch.Generator
with exactly the calls the reference makes (so a given seed selects the same random stream).

Order of operations is the reference's: the conditional forward sees the ids BEFORE the text step of that iteration,
the unconditional forwards see them AFTER it (parallel_generator.py:178, :217, :243-264), hence they are separate
forwards. The uncond_text forward is skipped when cfg_scale == 0 (its logits are unused there, :286-287).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .. import _lib
from .._lib import check, lib, ptr, stream_ptr
from ..schedule import (cosine_schedule, get_num_transfer_tokens as _num_transfer_row, image_generation_step_indices,
                        scheduled_mask_len)

MASK_TOKEN = 126336
NEW_LINE = 126084
# limits of the single-CTA re-mask / commit kernels and of the per-row image kernel (csrc/sampling.cu)
MAX_VQ_TOKENS, MAX_TEXT_TOKENS, MAX_CODEBOOK = 4096, 4096, 8192

__all__ = ["generate_ti2ti", "cosine_schedule", "get_num_transfer_tokens", "add_gumbel_noise", "mask_by_random_topk"]


def get_num_transfer_tokens(text_masked_indices: torch.Tensor, text_steps: int) -> torch.Tensor:
    """Same contract as the reference helper (:78-99): bool [B, T] -> int64 [B, text_steps]."""
    counts = text_masked_indices.sum(dim=1).tolist()
    return torch.tensor([_num_transfer_row(int(c), text_steps) for c in counts], dtype=torch.long,
                        device=text_masked_indices.device)


def add_gumbel_noise(logits, temperature=1.0, generator=None):  # pragma: no cover - fused into mmdp_text_step
    raise NotImplementedError("fused into the text-step kernel (mmdp_text_step); see generate_ti2ti")


def mask_by_random_topk(mask_len, probs, temperature=1.0, generator=None):  # pragma: no cover
    raise NotImplementedError("fused into the image-step kernel (mmdp_image_step); see generate_ti2ti")


class _Noise:
    """Draws the reference's random tensors from the caller's generator (same calls, same order), on the generator's
    device, and hands them to the kernels as device tensors."""

    def __init__(self, generator: Optional[torch.Generator], device: torch.device):
        self.g = generator
        self.dev = device
        self.gdev = generator.device if generator is not None else device

    def _to(self, t):
        return t if t.device == self.dev else t.to(self.dev, non_blocking=False)

    def rand(self, shape):
        return self._to(torch.rand(shape, dtype=torch.bfloat16, device=self.gdev, generator=self.g))

    def exponential(self, shape):
        return self._to(torch.empty(shape, dtype=torch.bfloat16, device=self.gdev).exponential_(1, generator=self.g))

    def randn(self, shape):
        return self._to(torch.randn(shape, dtype=torch.bfloat16, device=self.gdev, generator=self.g))


class DenoiseState:
    """Device-resident state of one generate_ti2ti call (ids, position maps, logits/workspace buffers)."""

    def __init__(self, model, ids_host: torch.Tensor, text_start: int, text_end: int, image_start: int, seq_len: int,
                 newline_every: int, uncon_text, uncon_image, cfg_scale: float, cfg_img: float, codebook_size: int):
        device = model.device
        self.model = model
        self.L = ids_host.shape[1]
        # limits of the sampling kernels (csrc/sampling.cu), checked before any forward runs
        if seq_len > MAX_VQ_TOKENS or text_end - text_start > MAX_TEXT_TOKENS:
            raise ValueError(f"at most {MAX_VQ_TOKENS} VQ tokens and {MAX_TEXT_TOKENS} text positions are supported "
                             f"(got {seq_len} / {text_end - text_start})")
        if codebook_size > MAX_CODEBOOK or codebook_size % 8:
            raise ValueError(f"codebook_size must be a multiple of 8 and <= {MAX_CODEBOOK} (got {codebook_size})")
        total_image_len = seq_len + seq_len // newline_every
        image_end = image_start + total_image_len
        self.text_start, self.text_end, self.seq_len = text_start, text_end, seq_len
        self.n_text = text_end - text_start
        self.total_masks = int((ids_host[0, text_start:text_end] == MASK_TOKEN).sum())
        self.pos_list = [i for i in range(image_start, image_end) if int(ids_host[0, i]) != NEW_LINE]   # :164-167
        assert len(self.pos_list) == seq_len, f"Expected {seq_len} VQ tokens, got {len(self.pos_list)}"
        # one pinned staging buffer -> one H2D copy for everything the loop needs from the host
        self.ids = ids_host.to(device, non_blocking=False).clone().contiguous()                       # combined_input_ids (:140)
        self.text_rows = torch.arange(text_start, text_end, dtype=torch.int32, device=device)
        self.pos = torch.tensor(self.pos_list, dtype=torch.int32, device=device)
        # row windows of the last transformer block (model.forward_rows): only rows whose logits are read need its output. Long
        # sequences only - short ones are launch-bound and the tiny parity models keep one fixed kernel schedule.
        img_lo, img_hi = min(self.pos_list), max(self.pos_list) + 1
        use = ids_host.shape[0] == 1 and ids_host.shape[1] >= 1024
        self.win_text = (text_start, text_end) if use else None
        self.win_img = (img_lo, img_hi) if use else None
        self.win_both = (min(text_start, img_lo), max(text_end, img_hi)) if use else None
        self.use_uncond = (cfg_scale > 0.0 and uncon_text is not None) or (cfg_img > 0.0 and uncon_image is not None)
        self.unc_t_ids = uncon_text.to(device=device, dtype=torch.int64) if uncon_text is not None else None
        self.unc_i_ids = uncon_image.to(device=device, dtype=torch.int64) if uncon_image is not None else None
        V = model.vocab_rows
        bf = dict(dtype=torch.bfloat16, device=device)
        self.text_logits = torch.empty((self.n_text, V), **bf)
        self.cond_vq = torch.empty((seq_len, codebook_size), **bf)
        self.unc_t_vq = torch.empty_like(self.cond_vq) if (self.use_uncond and cfg_scale != 0.0) else None
        self.unc_i_vq = torch.empty_like(self.cond_vq) if (self.use_uncond and cfg_img != 0.0) else None
        self.zeros_vq = torch.zeros_like(self.cond_vq) if (not self.use_uncond and (cfg_scale != 0.0 or cfg_img != 0.0)) else None
        self.x0_ws = torch.empty(self.n_text, dtype=torch.int64, device=device)
        self.conf_ws = torch.empty(self.n_text, dtype=torch.float64, device=device)
        self.sampled_ws = torch.empty(seq_len, dtype=torch.int32, device=device)
        self.selp_ws = torch.empty(seq_len, dtype=torch.float32, device=device)
        self.unk_ws = torch.empty(seq_len, dtype=torch.uint8, device=device)
        self.scratch_ids = torch.empty_like(self.ids)

    def bytes_h2d(self) -> int:
        n = self.ids.numel() * 8
        n += self.unc_t_ids.numel() * 8 if self.unc_t_ids is not None else 0
        n += self.unc_i_ids.numel() * 8 if self.unc_i_ids is not None else 0
        return n


def _window(model, win):
    """forward_rows keyword for the last-block row window, for models that take it (the tensor-parallel model does not)."""
    return {"row_window": win} if (win is not None and getattr(model, "supports_row_window", False)) else {}


def denoise_step(st: DenoiseState, step: int, is_img: bool, k_transfer: int, noise: "_Noise", text_steps: int,
                 temperature: float, text_temperature: float, cfg_scale: float, cfg_img: float, noise_schedule,
                 text_vocab_size: int, codebook_size: int, _trace: Optional[list] = None, text_masks_left: int = 1) -> None:
    """One iteration of the step loop (parallel_generator.py:177-344; the preview loop app.py:177-305 runs the same body)
    on device-resident state. No host<->device synchronisation happens in here.
    `text_masks_left` is the number of masked text positions entering this step (known on the host without a read-back:
    total - sum of the transfer counts so far); at 0 the reference skips the whole text step INCLUDING its Gumbel draw
    (`if text_masked_indices.sum() > 0`, :183), so no generator state is consumed here either.
    The forwards are issued here; the sampling halves (`text_sample`, `image_sample`) are shared with the packed batch loop
    (generators/batch.py)."""
    model, ids = st.model, st.ids
    # ---- conditional forward (:178): text rows x V, and the image rows x codebook window on image steps
    model.forward_rows(ids, rows_a=st.text_rows, out_a=st.text_logits, rows_b=st.pos if is_img else None,
                       col0_b=text_vocab_size, ncols_b=codebook_size, out_b=st.cond_vq if is_img else None,
                       **_window(model, st.win_both if is_img else st.win_text))
    text_sample(st, step, k_transfer, noise, text_temperature, _trace, text_masks_left)
    if not is_img:
        return
    # ---- unconditional forwards (:243-264) on the ids after the text step
    for out_name, prefix in uncond_inputs(st, cfg_scale, cfg_img):
        st.scratch_ids.copy_(ids)
        if prefix is not None:
            st.scratch_ids[:, : prefix.shape[1]] = prefix
        model.forward_rows(st.scratch_ids, rows_b=st.pos, col0_b=text_vocab_size, ncols_b=codebook_size,
                           out_b=getattr(st, out_name), **_window(model, st.win_img))
    image_sample(st, step, noise, text_steps, temperature, cfg_scale, cfg_img, noise_schedule, text_vocab_size, codebook_size,
                 _trace)


def text_sample(st: DenoiseState, step: int, k_transfer: int, noise: "_Noise", text_temperature: float,
                _trace: Optional[list] = None, text_masks_left: int = 1) -> None:
    """Text step (:181-217) on the conditional text logits in `st.text_logits`, guarded like the reference's `.sum() > 0` (:183)."""
    ids, V, n_text = st.ids, st.model.vocab_rows, st.n_text
    if text_masks_left > 0:
        un = noise.rand((1, n_text, V))[0] if text_temperature != 0 else None
        check(lib.mmdp_text_step(ptr(st.text_logits), None, V, n_text, V, 0.0, ptr(un), V, float(text_temperature),
                                 ids.data_ptr() + st.text_start * 8, MASK_TOKEN, int(k_transfer), ptr(st.x0_ws), ptr(st.conf_ws),
                                 stream_ptr()))
    if _trace is not None:
        _trace.append({"step": step, "ids_after_text": ids[0].clone()})


def uncond_inputs(st: DenoiseState, cfg_scale: float, cfg_img: float) -> list:
    """The unconditional forwards of an image step (:243-264), in the reference's order: [(name of the DenoiseState buffer that
    receives the image-row logits, prefix ids [1, n] that replace the start of the sequence, or None)]. Each runs on the ids
    after the text step with the prefix written over them; its length is the sequence's."""
    if not st.use_uncond:
        return []
    out = []
    if cfg_scale != 0.0:
        out.append(("unc_t_vq", st.unc_t_ids))
    if cfg_img != 0.0:
        out.append(("unc_i_vq", st.unc_i_ids))
    return out


def image_sample(st: DenoiseState, step: int, noise: "_Noise", text_steps: int, temperature: float, cfg_scale: float,
                 cfg_img: float, noise_schedule, text_vocab_size: int, codebook_size: int, _trace: Optional[list] = None) -> None:
    """Image step (:220-344) on the logits in `st.cond_vq` and the unconditional buffers named by `uncond_inputs`."""
    ids, seq_len = st.ids, st.seq_len
    ua = ub = None
    if st.use_uncond:
        ua = st.unc_t_vq if cfg_scale != 0.0 else None
        ub = st.unc_i_vq if cfg_img != 0.0 else None
    elif st.zeros_vq is not None:
        # no uncond inputs: the reference mixes against zeros (:277-278)
        ua = st.zeros_vq if cfg_scale != 0.0 else None
        ub = st.zeros_vq if cfg_img != 0.0 else None
    q = noise.exponential((seq_len, codebook_size)) if temperature != 0 else None   # torch.multinomial's draw (:299-302)
    ratio = 1.0 * (step + 1) / text_steps
    img_temp = temperature * (1.0 - ratio)                                           # :330
    rn = noise.randn((1, seq_len))                                                   # mask_by_random_topk (:30-31)
    check(lib.mmdp_image_step(0, ptr(st.cond_vq), ptr(ua), ptr(ub), codebook_size, seq_len, codebook_size,
                              float(cfg_scale), float(cfg_img), ptr(q), ptr(rn), float(img_temp),
                              scheduled_mask_len(seq_len, step, text_steps, noise_schedule), ptr(ids), ptr(st.pos),
                              MASK_TOKEN, text_vocab_size, ptr(st.sampled_ws), ptr(st.selp_ws), ptr(st.unk_ws), None,
                              None, None, stream_ptr()))
    if _trace is not None:
        _trace[-1].update(sampled=st.sampled_ws.clone(), ids_after_image=ids[0].clone())


def denoise_loop(st: DenoiseState, text_steps: int, timesteps: int, temperature: float, text_temperature: float,
                 cfg_scale: float, cfg_img: float, noise_schedule, generator, text_vocab_size: int, codebook_size: int,
                 _trace: Optional[list] = None) -> torch.Tensor:
    """The hot loop (parallel_generator.py:174-344) on device-resident state; returns the id buffer (device).
    No host<->device synchronisation happens in here."""
    num_transfer = _num_transfer_row(st.total_masks, text_steps)                              # :153-154
    img_steps = set(image_generation_step_indices(text_steps, timesteps))                     # :157-159
    noise = _Noise(generator, st.model.device)
    masks_left = st.total_masks
    for step in range(text_steps):
        denoise_step(st, step, step in img_steps, num_transfer[step], noise, text_steps, temperature, text_temperature,
                     cfg_scale, cfg_img, noise_schedule, text_vocab_size, codebook_size, _trace, text_masks_left=masks_left)
        masks_left -= num_transfer[step]
    return st.ids


@torch.no_grad()
def generate_ti2ti(
    model,
    input_ids,
    text_start,
    text_end,
    image_start,
    seq_len,
    newline_every,
    text_steps=100,
    text_gen_length=256,
    text_block_length=64,
    timesteps=100,
    temperature=1.0,
    text_temperature=0.7,
    cfg_scale=0.0,
    cfg_img=4.0,
    uncon_text=None,
    uncon_image=None,
    tokenizer=None,
    remasking="low_confidence",
    noise_schedule=cosine_schedule,
    generator=None,
    text_vocab_size=126356,
    codebook_size=8192,
    _trace: Optional[list] = None,
):
    """Joint text+image mask-predict generation. Arguments, defaults, side effects (input_ids is not modified) and
    return value `(List[int] image VQ tokens, str | List[int] text)` are those of the reference function."""
    check_request(model, input_ids, remasking)
    ids_host = input_ids.detach().to("cpu", torch.int64)
    total_image_len = seq_len + seq_len // newline_every
    print(f"Interleaved generation: {text_steps} total steps")
    print(f"  - Text generation range: [{text_start}, {text_end})")
    print(f"  - Image generation range: [{image_start}, {image_start + total_image_len}) (total {total_image_len} including newlines)")
    print(f"  - VQ tokens: {seq_len}")
    st = DenoiseState(model, ids_host, text_start, text_end, image_start, seq_len, newline_every, uncon_text, uncon_image,
                      cfg_scale, cfg_img, codebook_size)
    ids = denoise_loop(st, text_steps, timesteps, temperature, text_temperature, cfg_scale, cfg_img, noise_schedule,
                       generator, text_vocab_size, codebook_size, _trace)

    # ---- extract results (:346-368): the only device->host read of the call
    final = ids[0].cpu()
    if hasattr(model, "raise_device_errors"):
        model.raise_device_errors()   # e.g. a token id outside the vocabulary: IndexError, like nn.Embedding in the reference
    image_tokens, generated_text, n_text_tokens = extract_results(st, final, tokenizer, text_vocab_size, codebook_size)
    print("Interleaved generation complete.")
    print(f"  - Generated text: {n_text_tokens} tokens")
    print(f"  - Generated image: {len(image_tokens)} VQ tokens (range [0, {codebook_size}))")
    return image_tokens, generated_text


def check_request(model, input_ids, remasking) -> None:
    """The argument checks generate_ti2ti makes before it builds its state, in its order."""
    if remasking != "low_confidence":
        # 'random' requests int64 uniform noise in the reference and raises there too (:195-197)
        raise NotImplementedError(remasking)
    if not hasattr(model, "forward_rows"):
        raise TypeError("generate_ti2ti needs a mmada_parallel_b200.model.LLaDAForMultiModalGeneration (H100-native) model")
    if input_ids.shape[0] != 1:
        raise ValueError("the image path of generate_ti2ti is single-sample (reference :224/:340 read batch row 0 only)")


def extract_results(st: DenoiseState, final: torch.Tensor, tokenizer, text_vocab_size: int, codebook_size: int):
    """(:346-368) The image VQ tokens and the text of the final id row `final` (host). Image tokens still masked are drawn
    from the GLOBAL CPU RNG like the reference (:362). Returns (image tokens, text, number of text tokens)."""
    text_tokens = [t for t in final[st.text_start:st.text_end].tolist() if t != MASK_TOKEN]
    generated_text = tokenizer.decode(text_tokens, skip_special_tokens=True) if tokenizer is not None else text_tokens
    image_tokens: List[int] = []
    for t in final[torch.tensor(st.pos_list)].tolist():
        if t != MASK_TOKEN:
            image_tokens.append(max(0, min(t - text_vocab_size, codebook_size - 1)))
        else:
            image_tokens.append(int(torch.randint(0, codebook_size, (1,)).item()))
    return image_tokens, generated_text, len(text_tokens)
