"""Drop-in for the variant-M model object: `MMadaModelLM.interleave_generate`
(MMaDA-Parallel-M/models/modeling_mmada.py:118-248) and `MMadaModelLM.mmu_generate` (:619-691, SURVEY 8f rank 3, the
generation mode M's validation loop calls) on top of the same native forward.

Differences from variant A that are preserved here (SURVEY.md Appendix A 10-11):
  * one forward per step over the CFG batch [cond; uncond] (B = 2), never B = 1 (:168-177);
  * text logits are CFG-mixed: cond + text_cfg * (uncond - cond) (:179), argmax + fp64 softmax confidence on the mix;
  * image logits are (1 + s) * cond - s * uncond (:216), ALWAYS sampled with torch.multinomial (:222);
  * re-masking uses Gumbel noise and a strict `<` cut-off against the k-th smallest confidence (M/models/sampling.py:31-36);
  * returns the sampled ids BEFORE re-masking and the text span, as tensors (:244-248).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch

from ._lib import check, lib, ptr, stream_ptr
from .generators.parallel_generator import _Noise
from .model import LLaDAForMultiModalGeneration
from .schedule import cosine_schedule, get_num_transfer_tokens_m, image_generation_step_indices, scheduled_mask_len


class MMadaModelLM(LLaDAForMultiModalGeneration):
    def __init__(self, config, max_seq_len: Optional[int] = None, max_batch: int = 2, device: str = "cuda:0",
                 precision: str = "bf16"):
        super().__init__(config, max_seq_len=max_seq_len, max_batch=max(2, max_batch), device=device, precision=precision)

    def forward(self, input_ids=None, **kw):
        """M calls the backbone directly: `self(ids).logits` (modeling_mmada.py:172)."""
        kw.pop("infer", None)
        return super().forward(input_ids, infer=True, **kw)

    __call__ = forward

    @torch.no_grad()
    def interleave_generate(
        self,
        input_ids: torch.LongTensor = None,
        uncond_input_ids: torch.LongTensor = None,
        text_cfg: float = 0.0,
        image_cfg: float = 3.5,
        noise_schedule: Callable = cosine_schedule,
        text_steps: int = 100,
        image_steps: int = 100,
        reserved_token_mapping: Dict = None,
        generator: torch.Generator = None,
        config=None,
        remasking="low_confidence",
        text_temperature: float = 0.0,
        image_temperature: float = 1.0,
        **kwargs,
    ):
        st = InterleaveState(self, input_ids, uncond_input_ids, text_cfg, image_cfg, noise_schedule, text_steps, image_steps,
                             reserved_token_mapping, generator, config, remasking, text_temperature, image_temperature, **kwargs)
        for i in range(text_steps):
            is_img = i in st.img_idx
            self.forward_rows(st.both, rows_a=st.rows_text, out_a=st.text_logits, rows_b=st.rows_img if is_img else None,
                              col0_b=st.tvoc, ncols_b=st.C, out_b=st.img_logits if is_img else None,
                              row_window=st.window(i))                                           # :172
            interleave_text_step(st, i, st.text_logits[:st.max_seq], st.text_logits[st.max_seq:])
            if is_img:
                interleave_image_step(st, i, st.img_logits[:st.n_vq], st.img_logits[st.n_vq:])
        return st.results()

    @torch.no_grad()
    def mmu_generate(self, idx=None, input_embeddings=None, max_new_tokens=128, steps=128, block_length=128, temperature=0.0,
                     top_k=None, eot_token=None, cfg_scale=0.0, remasking="low_confidence", mask_id=126336,
                     attention_mask=None):
        """Block-wise (semi-autoregressive) un-masking of `max_new_tokens` masks appended to the prompt `idx [B, P]`
        (modeling_mmada.py:619-691); returns x [B, P + max_new_tokens] on the model device. Per step one forward over
        [x] (or the CFG batch [x; x with its prompt masked]) restricted to the current block's rows, then the text-step
        kernel per batch row: logits = un + (cfg + 1) * (l - un) in bf16 (:660), argmax, fp64 softmax confidence, the k
        most confident masked positions committed (:676-683). Positions after the block carry confidence -inf in the
        reference (:673) and earlier blocks are complete, so only the block's rows are evaluated.
        `attention_mask`: the reference turns a mask with zeros into an `attention_bias` (:626-627) that the M backbone never
        reads (its blocks take `attention_mask`, which stays None) - padding is NOT masked there, so the argument is accepted
        and has no effect (pinned against the real reference in oracle/make_golden_m_modes.py).
        `temperature > 0`: fp64 Gumbel-max (:49-60); the uniform noise has the FULL logits shape [B', L, V] and comes from the
        global RNG of the logits' device, drawn here with the same call (same stream as the reference on a GPU).
        Not built (raise): `remasking='random'` (global RNG), `input_embeddings`."""
        if idx is None or input_embeddings is not None:
            raise NotImplementedError("mmu_generate: only token-id prompts (idx) are supported")
        if remasking != "low_confidence":
            raise NotImplementedError(remasking)
        dev = self.device
        idx = idx.to(device=dev, dtype=torch.int64)
        B, P = idx.shape
        if bool((idx == mask_id).any()):
            raise ValueError("mmu_generate: the prompt must not contain mask tokens")
        assert max_new_tokens % block_length == 0                                              # :642
        num_blocks = max_new_tokens // block_length
        assert steps % num_blocks == 0                                                         # :645
        steps = steps // num_blocks
        L = P + max_new_tokens
        use_cfg = cfg_scale > 0.0
        nb = 2 * B if use_cfg else B
        both = torch.full((nb, L), int(mask_id), dtype=torch.int64, device=dev)              # rows [x; un_x]
        both[:B, :P] = idx                                                                     # un_x: prompt stays masked (:656)
        V = self.vocab_rows
        text_logits = torch.empty((nb * block_length, V), dtype=torch.bfloat16, device=dev)
        x0_ws = torch.empty(block_length, dtype=torch.int64, device=dev)
        conf_ws = torch.empty(block_length, dtype=torch.float64, device=dev)
        num_transfer = get_num_transfer_tokens_m(block_length, steps)                          # every block starts all-masked
        for blk in range(num_blocks):
            bs = P + blk * block_length
            rows = torch.cat([torch.arange(r * L + bs, r * L + bs + block_length, dtype=torch.int32, device=dev)
                              for r in range(nb)])
            for i in range(steps):
                self.forward_rows(both, rows_a=rows, out_a=text_logits)
                u64 = None
                if temperature != 0:
                    # rand_like(logits [B, L, V], dtype=float64): the whole sequence's noise is drawn (keeps the RNG stream
                    # aligned with the reference); only the current block's rows are read by the kernel
                    u64 = (self._mmu_noise(blk * steps + i, (B, L, V)) if getattr(self, "_mmu_noise", None) is not None
                           else torch.rand((B, L, V), dtype=torch.float64, device=dev)).to(dev).contiguous()
                for j in range(B):
                    cond = text_logits.data_ptr() + j * block_length * V * 2
                    unc = text_logits.data_ptr() + (B + j) * block_length * V * 2 if use_cfg else None
                    # kernel: c + cfg * (u - c) with c = un-logits, u = cond logits, cfg = cfg_scale + 1
                    a0, a1, cf = (unc, cond, float(cfg_scale + 1)) if use_cfg else (cond, None, 0.0)
                    ids_ptr = both.data_ptr() + (j * L + bs) * 8
                    if u64 is not None:
                        check(lib.mmdp_text_step_gumbel64(a0, a1, V, block_length, V, cf, u64.data_ptr() + (j * L + bs) * V * 8, V,
                                                          float(temperature), ids_ptr, int(mask_id), int(num_transfer[i]),
                                                          ptr(x0_ws), ptr(conf_ws), stream_ptr()))
                    else:
                        check(lib.mmdp_text_step(a0, a1, V, block_length, V, cf, None, 0, 0.0, ids_ptr, int(mask_id),
                                                 int(num_transfer[i]), ptr(x0_ws), ptr(conf_ws), stream_ptr()))
                if use_cfg:
                    both[B:, P:] = both[:B, P:]
        return both[:B].clone()

    @torch.no_grad()
    def t2i_generate(
        self,
        input_ids: torch.LongTensor = None,
        uncond_input_ids: torch.LongTensor = None,
        attention_mask=None,
        uncond_attention_mask=None,
        temperature=1.0,
        timesteps=18,
        guidance_scale=0,
        noise_schedule=cosine_schedule,
        generator: torch.Generator = None,
        config=None,
        seq_len=1024,
        mask_token_id=126336,
        resolution=512,
        codebook_size=8192,
        **kwargs,
    ):
        """MaskGit text-to-image decoding of variant M (modeling_mmada.py:265-359): the last seq_len + 1 positions of
        `input_ids [B, L]` hold the image tokens followed by one closing token. Per step: one forward over [input_ids] or, with
        guidance, over the batch [input_ids; uncond_prefix + input_ids[:, resolution + 1:]] with the LM head restricted to the
        image rows x the codebook window; then per batch row the variant-M image-step kernel (CFG mix (1 + s) c - s u, softmax,
        torch.multinomial's exponential race, confidence, Gumbel re-mask with the strict cut-off). Kept from the reference:
        `input_ids` is updated IN PLACE (:355); `temperature` is multiplied by (1 - ratio) on every step, i.e. it compounds
        (:352); the attention masks only build an attention_bias the backbone never reads (no effect; pinned in
        oracle/make_golden_m_modes.py). Returns the last step's sampled ids [B, seq_len] (before re-masking)."""
        uni_prompting = kwargs.get("uni_prompting", None)
        dev = self.device
        n, C = int(seq_len), int(codebook_size)
        tvoc = len(uni_prompting.text_tokenizer)
        caller_ids = input_ids
        ids = input_ids.to(device=dev, dtype=torch.int64).clone().contiguous()
        B, L = ids.shape
        use_cfg = uncond_input_ids is not None and guidance_scale > 0
        nb = 2 * B if use_cfg else B
        if nb > self.max_batch:
            raise ValueError(f"t2i_generate: batch {nb} (incl. the guidance copy) exceeds the model's max_batch={self.max_batch}")
        both = torch.empty((nb, L), dtype=torch.int64, device=dev)
        if use_cfg:
            unc_prefix = uncond_input_ids.to(device=dev, dtype=torch.int64)[:, : resolution + 1]           # :298
            if unc_prefix.shape[1] != resolution + 1 or unc_prefix.shape[0] != B:
                raise ValueError("t2i_generate: uncond_input_ids must be [B, >= resolution + 1]")
        p0 = L - (n + 1)
        pos = torch.arange(p0, p0 + n, dtype=torch.int32, device=dev)
        rows = torch.cat([pos + r * L for r in range(nb)])
        logits = torch.empty((nb * n, C), dtype=torch.bfloat16, device=dev)
        sampled_ws = torch.zeros((B, n), dtype=torch.int32, device=dev)
        selp_ws = torch.empty(n, dtype=torch.float32, device=dev)
        unk_ws = torch.empty(n, dtype=torch.uint8, device=dev)
        noise = _Noise(generator, dev)
        for step in range(timesteps):
            both[:B] = ids
            if use_cfg:
                both[B:, : resolution + 1] = unc_prefix                                                    # :304-305
                both[B:, resolution + 1:] = ids[:, resolution + 1:]
            self.forward_rows(both, rows_b=rows, col0_b=tvoc, ncols_b=C, out_b=logits)                     # :309 / :319
            q = noise.exponential((B * n, C))                                                              # multinomial over [B*n, C] (:327)
            ratio = 1.0 * (step + 1) / timesteps
            temperature = temperature * (1.0 - ratio)                                                      # :352 (compounds)
            un = torch.zeros((B, n), dtype=torch.bfloat16, device=noise.gdev).uniform_(0, 1, generator=generator).to(dev)
            for b in range(B):
                cond = logits.data_ptr() + b * n * C * 2
                # no guidance: (1 + 0) * cond - 0 * cond == cond in bf16, the kernel's variant-M mix with itself as "uncond"
                unc = logits.data_ptr() + (B + b) * n * C * 2 if use_cfg else cond
                s = float(guidance_scale) if use_cfg else 0.0
                check(lib.mmdp_image_step(1, cond, unc, None, C, n, C, s, float(1 + s), q.data_ptr() + b * n * C * 2,
                                          un.data_ptr() + b * n * 2, float(temperature),
                                          scheduled_mask_len(n, step, timesteps, noise_schedule), ids.data_ptr() + b * L * 8,
                                          ptr(pos), int(mask_token_id), tvoc, sampled_ws.data_ptr() + b * n * 4, ptr(selp_ws),
                                          ptr(unk_ws), None, None, None, stream_ptr()))
        if torch.is_tensor(caller_ids):
            caller_ids.copy_(ids.to(caller_ids.device))                                                    # in-place update, like the reference
        self.raise_device_errors()
        return sampled_ws.to(torch.int64)


def interleave_layout(config, uni_prompting, input_ids, uncond_input_ids, text_steps: int, image_steps: int) -> dict:
    """Host-side shape of one interleave_generate request, checked before anything touches the device: prompt length P, sequence
    length L = P + num_vq_tokens + max_seq_length + 2, text start t0, text vocabulary size and codebook size."""
    n_vq = int(config.model.mmada.num_vq_tokens)
    max_seq = int(config.dataset.preprocessing.max_seq_length)
    P = int(input_ids.shape[-1])
    if int(uncond_input_ids.shape[-1]) != P:
        raise ValueError("cond and uncond prompts must have equal length (padding is not masked, SURVEY App. A3)")
    L = P + n_vq + max_seq + 2                                                                   # soi, vq, eoi, bos, text masks
    return dict(n_vq=n_vq, max_seq=max_seq, P=P, L=L, t0=L - max_seq, C=int(config.model.mmada.codebook_size),
                tvoc=len(uni_prompting.text_tokenizer),
                img_idx=set(image_generation_step_indices(text_steps, image_steps)))


class InterleaveState:
    """Device-resident state of one interleave_generate request (modeling_mmada.py:118-248): the CFG id buffer [cond; uncond],
    its logits rows, the sampling workspaces and the request's noise source. `interleave_generate` and
    generators/batch.py::interleave_generate_batch advance it with `interleave_text_step` / `interleave_image_step`."""

    def __init__(self, model, input_ids, uncond_input_ids, text_cfg, image_cfg, noise_schedule, text_steps, image_steps,
                 reserved_token_mapping, generator, config, remasking, text_temperature, image_temperature, **kwargs):
        if not (text_cfg or image_cfg):
            raise ValueError("text_cfg and image_cfg cannot be both 0")                      # :181-182
        if remasking != "low_confidence":
            raise NotImplementedError(remasking)
        uni_prompting = kwargs.get("uni_prompting", None)
        self._text_noise = kwargs.get("_text_noise", None)  # tests: injects the fp64 uniform noise instead of the global-RNG draw
        lay = interleave_layout(config, uni_prompting, input_ids, uncond_input_ids, text_steps, image_steps)
        self.n_vq, self.max_seq, self.C, self.tvoc, self.img_idx = lay["n_vq"], lay["max_seq"], lay["C"], lay["tvoc"], lay["img_idx"]
        self.text_cfg, self.image_cfg, self.noise_schedule = float(text_cfg), float(image_cfg), noise_schedule
        self.text_steps, self.text_temperature, self.image_temperature = text_steps, text_temperature, image_temperature
        self.generator = generator
        dev = self.dev = model.device
        self.mask_id = mask_id = int(model.config.mask_token_id)
        n_vq, max_seq = self.n_vq, self.max_seq
        inp = input_ids.to(device=dev, dtype=torch.int64).unsqueeze(0)
        unc = uncond_input_ids.to(device=dev, dtype=torch.int64).unsqueeze(0)
        full = lambda n, v: torch.full((1, n), int(v), dtype=torch.int64, device=dev)
        out_ids = torch.cat([full(1, reserved_token_mapping["<|soi|>"]), full(n_vq, mask_id),
                             full(1, reserved_token_mapping["<|eoi|>"]), full(1, uni_prompting.text_tokenizer.bos_token_id),
                             full(max_seq - 1, mask_id)], dim=1)                               # :142-148
        P = self.P = inp.shape[1]
        L = self.L = P + out_ids.shape[1]
        both = self.both = torch.empty((2, L), dtype=torch.int64, device=dev)                  # [cond; uncond] id buffer
        both[0, :P] = inp[0]
        both[1, :P] = unc[0]
        both[:, P:] = out_ids
        self.num_transfer = get_num_transfer_tokens_m(max_seq - 1, text_steps)                # bos is not a mask
        V = model.vocab_rows
        t0 = self.t0 = L - max_seq
        self.rows_text = torch.cat([torch.arange(t0, L, dtype=torch.int32, device=dev),
                                    torch.arange(L + t0, 2 * L, dtype=torch.int32, device=dev)])
        self.pos = torch.arange(P + 1, P + 1 + n_vq, dtype=torch.int32, device=dev)
        self.rows_img = torch.cat([self.pos, self.pos + L])
        self.text_logits = torch.empty((2 * max_seq, V), dtype=torch.bfloat16, device=dev)
        self.img_logits = torch.empty((2 * n_vq, self.C), dtype=torch.bfloat16, device=dev)
        self.x0_ws = torch.empty(max_seq, dtype=torch.int64, device=dev)
        self.conf_ws = torch.empty(max_seq, dtype=torch.float64, device=dev)
        self.sampled_ws = torch.zeros(n_vq, dtype=torch.int32, device=dev)
        self.selp_ws = torch.empty(n_vq, dtype=torch.float32, device=dev)
        self.unk_ws = torch.empty(n_vq, dtype=torch.uint8, device=dev)
        self.noise = _Noise(generator, dev)
        self.any_image_step = False
        # positions whose logits are read, per batch row: the last block computes its attention output / MLP for them only
        # (model.forward_rows, row_window; long sequences only - the tiny parity models keep one fixed kernel schedule)
        self.win_text, self.win_img = ((t0, L), (P + 1, L)) if L >= 1024 else (None, None)

    def window(self, i: int):
        """The last-block row window of step i (per sequence): the text rows, and on image steps the image rows too."""
        return self.win_img if i in self.img_idx else self.win_text

    def results(self):
        if not self.any_image_step:
            raise RuntimeError("no image step was scheduled (the reference would hit an undefined `sampled_ids`)")
        return_image_ids = self.sampled_ws.to(torch.int64).unsqueeze(0)
        return_text_ids = self.both[0:1, -self.max_seq:].clone()
        return return_image_ids, return_text_ids


def interleave_text_step(st: InterleaveState, i: int, cond: torch.Tensor, uncond: torch.Tensor) -> None:
    """Step i's text step on the CFG-mixed logits (:179-209): cond / uncond [max_seq, V] are the text rows' logits of the two
    sequences. Only the cond row's ids change; the uncond row then shares the generated suffix (:166-169)."""
    max_seq, V = st.max_seq, cond.shape[1]
    if st.text_temperature != 0:
        # add_gumbel_noise (:49-60): fp64 uniform noise of the text-logits shape from the GLOBAL RNG of the logits'
        # device - the same call the reference makes on a GPU, so the same Philox stream is consumed
        u64 = (st._text_noise(i, (1, max_seq, V)) if st._text_noise is not None
               else torch.rand((1, max_seq, V), dtype=torch.float64, device=st.dev)).to(st.dev).contiguous()
        check(lib.mmdp_text_step_gumbel64(ptr(cond), ptr(uncond), V, max_seq, V, st.text_cfg, ptr(u64), V,
                                          float(st.text_temperature), st.both.data_ptr() + st.t0 * 8, st.mask_id,
                                          int(st.num_transfer[i]), ptr(st.x0_ws), ptr(st.conf_ws), stream_ptr()))
    else:
        check(lib.mmdp_text_step(ptr(cond), ptr(uncond), V, max_seq, V, st.text_cfg, None, 0, 0.0,
                                 st.both.data_ptr() + st.t0 * 8, st.mask_id, int(st.num_transfer[i]), ptr(st.x0_ws),
                                 ptr(st.conf_ws), stream_ptr()))
    st.both[1, st.P:] = st.both[0, st.P:]


def interleave_image_step(st: InterleaveState, i: int, cond: torch.Tensor, uncond: torch.Tensor) -> None:
    """Step i's image step (:211-240) on cond / uncond [n_vq, codebook_size], the image rows' codebook logits; draws the
    multinomial's exponentials, then the re-masking noise, from the request's generator."""
    n_vq, C = st.n_vq, st.C
    st.any_image_step = True
    q = st.noise.exponential((n_vq, C))                                                         # multinomial (:222)
    ratio = 1.0 * (i + 1) / st.text_steps
    temp = st.image_temperature * (1.0 - ratio)                                                 # :236
    # gumbel_noise(): torch.zeros_like(t).uniform_(0, 1, generator=generator)  (M/models/sampling.py:14-15)
    un = torch.zeros((1, n_vq), dtype=torch.bfloat16, device=st.noise.gdev).uniform_(0, 1, generator=st.generator).to(st.dev)
    check(lib.mmdp_image_step(1, ptr(cond), ptr(uncond), None, C, n_vq, C, st.image_cfg, float(1 + st.image_cfg), ptr(q), ptr(un),
                              float(temp), scheduled_mask_len(n_vq, i, st.text_steps, st.noise_schedule), ptr(st.both),
                              ptr(st.pos), st.mask_id, st.tvoc, ptr(st.sampled_ws), ptr(st.selp_ws), ptr(st.unk_ws), None, None,
                              None, stream_ptr()))
    st.both[1, st.P:] = st.both[0, st.P:]
