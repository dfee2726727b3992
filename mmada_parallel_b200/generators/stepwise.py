"""Drop-in for the Gradio preview loop `generate_ti2ti_stepwise` (MMaDA-Parallel-A/app.py:143-398; SURVEY.md section 8f
rank 2): the same denoising step as generate_ti2ti (`denoise_step`, CUDA kernels behind the C ABI) driven as a Python
generator that yields `(step, text_display, image, status)` at the reference's cadence.

Differences to generate_ti2ti that the reference makes and this file keeps: image steps are
`linspace(0, T-1, int(0.3 T))` (:162-164), there is no `timesteps` argument, every image step decodes the PRE-remask
sample for the preview and greys out the cells that were re-masked (:307-335), and when no image step ran the final image
is decoded with `codebook_size // 2` in the masked cells (:352-396). Each yield reads the text span (and on image steps
the image cells) back to the host - the only synchronisation points.

`vqvae` is a native decoder (mmada_parallel_b200.magvit.MAGVITv2 protocol, see utils/image_utils.py). Deviations, stated:
`remasking` other than 'low_confidence' raises NotImplementedError (the reference's 'random' branch requests int64 uniform
noise when a generator is given and raises too; its catch-all `else` makes every confidence 1.0, leaving the choice to
torch.topk's unspecified tie order); a preview decode error is not swallowed.
"""
from __future__ import annotations

from typing import Optional

import torch

from ..schedule import cosine_schedule, get_num_transfer_tokens as _num_transfer_row, stepwise_image_step_indices
from ..utils.image_utils import decode_vq_to_image, overlay_masked_cells, vq_scale
from .parallel_generator import MASK_TOKEN, DenoiseState, _Noise, denoise_step


def decode_text_with_masks(combined_input_ids, text_start, text_end, tokenizer, mask_token) -> str:
    """app.py:102-140: the text span as a string; runs of mask tokens are drawn as blocks, long runs abbreviated."""
    def run(n):
        return "▓" * n if n <= 10 else f"▓▓▓▓▓[...{n - 5} more]"
    parts, masks = [], 0
    for t in combined_input_ids[0, text_start:text_end].cpu().tolist():
        if t == mask_token:
            masks += 1
            continue
        if masks > 0:
            parts.append(run(masks))
            masks = 0
        try:
            piece = tokenizer.decode([t], skip_special_tokens=False, clean_up_tokenization_spaces=False)
            if piece.strip() or piece in [" ", "\n", "\t"]:
                parts.append(piece)
        except Exception:                                                          # the reference uses a bare except (:131)
            parts.append(f"[{t}]")
    if masks > 0:
        parts.append(run(masks))
    return "".join(parts)


@torch.no_grad()
def generate_ti2ti_stepwise(
    model, input_ids, text_start, text_end, image_start, seq_len, newline_every,
    text_steps=100, temperature=1.0, text_temperature=0.7, cfg_scale=0.0, cfg_img=4.0,
    uncon_text=None, uncon_image=None, tokenizer=None, remasking="low_confidence",
    noise_schedule=cosine_schedule, generator=None, text_vocab_size=126356,
    codebook_size=8192, vqvae=None, image_height=512, image_width=512, _trace: Optional[list] = None,
):
    if remasking != "low_confidence":
        raise NotImplementedError(remasking)
    if not hasattr(model, "forward_rows"):
        raise TypeError("generate_ti2ti_stepwise needs a mmada_parallel_b200.model.LLaDAForMultiModalGeneration (H100-native) model")
    if input_ids.shape[0] != 1:
        raise ValueError("the image path is single-sample (the reference reads batch row 0 only, app.py:199/:300)")
    ids_host = input_ids.detach().to("cpu", torch.int64)
    st = DenoiseState(model, ids_host, text_start, text_end, image_start, seq_len, newline_every, uncon_text, uncon_image,
                      cfg_scale, cfg_img, codebook_size)
    num_transfer = _num_transfer_row(st.total_masks, text_steps)
    img_steps = set(stepwise_image_step_indices(text_steps))
    noise = _Noise(generator, model.device)
    ids = st.ids

    def preview(codes: torch.Tensor, masked_idx):
        img = decode_vq_to_image(codes, None, None, image_height, image_width, vqvae)
        if masked_idx:
            scale = vq_scale(vqvae)
            token_h, token_w = image_height // scale, image_width // scale
            img = overlay_masked_cells(img, masked_idx, token_w, image_height // token_h, image_width // token_w)
        return img

    last_image = None
    masks_left = st.total_masks
    yield 0, decode_text_with_masks(ids, text_start, text_end, tokenizer, MASK_TOKEN), None, f"Step 0/{text_steps}"
    for step in range(text_steps):
        is_img = step in img_steps
        denoise_step(st, step, is_img, num_transfer[step], noise, text_steps, temperature, text_temperature, cfg_scale,
                     cfg_img, noise_schedule, text_vocab_size, codebook_size, _trace, text_masks_left=masks_left)
        masks_left -= num_transfer[step]
        emit = step % 5 == 0 or is_img or step == text_steps - 1                                 # :345
        if not (emit or is_img):
            continue
        img_left = None
        if is_img:
            masked = (ids[0, st.pos.long()] == MASK_TOKEN)                                      # cells re-masked by this step
            img_left = int(masked.sum())
            last_image = preview(st.sampled_ws.long().unsqueeze(0), masked.nonzero().flatten().tolist())
        text_display = decode_text_with_masks(ids, text_start, text_end, tokenizer, MASK_TOKEN)
        remaining = int((ids[0, text_start:text_end] == MASK_TOKEN).sum())
        status = f"Step {step + 1}/{text_steps} | Text: {(1 - remaining / (text_end - text_start)) * 100:.1f}%"
        if is_img:
            status += f" | Image: {(1 - img_left / seq_len) * 100:.1f}%"
        yield step + 1, text_display, last_image, status
    final_text = decode_text_with_masks(ids, text_start, text_end, tokenizer, MASK_TOKEN)
    if last_image is None:                                                                       # :352-396
        tok = ids[0, st.pos.long()]
        masked = tok == MASK_TOKEN
        codes = torch.where(masked, torch.full_like(tok, codebook_size // 2),
                            torch.clamp(tok - text_vocab_size, 0, codebook_size - 1))
        last_image = preview(codes.unsqueeze(0), masked.nonzero().flatten().tolist())
    yield text_steps, final_text, last_image, "✓ Complete"
