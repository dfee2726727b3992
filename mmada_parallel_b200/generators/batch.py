"""Several generate_ti2ti requests on one GPU through packed forwards.

`generate_ti2ti_batch(model, requests)` returns exactly what `[generate_ti2ti(model, **r) for r in requests]` returns (ids, text,
the state of every request's generator afterwards). Requests may differ in every argument: prompt and length, grid
(seq_len / newline_every), text_steps, timesteps, temperatures, CFG scales, unconditional inputs, tokenizer.

Padding cannot batch them: the reference never masks padding (SDPA gets attn_mask=None), so a padded row computes something
else than the same request alone. A PACKED forward (model.forward_rows_packed) lays the sequences end to end instead; each is
computed as if it were alone. A global step advances every unfinished request by one of its own steps:
  1. one packed conditional forward over the active requests (text rows; image rows of those in an image step);
  2. each request's text step (`text_sample`, the code generate_ti2ti runs);
  3. one packed forward over the unconditional sequences of the requests in an image step (one or two per request, each of
     its request's length), after their text steps like in the reference;
  4. each request's image step (`image_sample`).
Requests with fewer steps drop out. A set of more than `max_batch` sequences runs as several packed forwards. The
tensor-parallel model (tensor_parallel.TensorParallelLLaDA) serves batches too: every rank calls generate_ti2ti_batch with the
same requests and generator seeds, as it calls generate_ti2ti.
The sampling stays per request: each draws from its own generator in the order generate_ti2ti does, so the draws of one
request do not depend on its neighbours. Still-masked image tokens are drawn from the global CPU RNG after the loop, in request
order, like sequential calls would.

`interleave_generate_batch(model, requests)` does the same for variant M's `MMadaModelLM.interleave_generate`: one packed forward
per global step over the cond and uncond sequences of every active request, then each request's text step and, on its image
steps, its image step (`interleave_text_step` / `interleave_image_step`, the code interleave_generate runs). Each sequence gets
the last-block row window interleave_generate would give it.
"""
from __future__ import annotations

import inspect
from typing import List, Sequence

import torch

from ..schedule import get_num_transfer_tokens, image_generation_step_indices
from .parallel_generator import (DenoiseState, _Noise, check_request, extract_results, generate_ti2ti, image_sample,
                                 text_sample, uncond_inputs)

__all__ = ["generate_ti2ti_batch", "interleave_generate_batch", "batch_schedule", "packed_chunks"]

_SIGNATURE = inspect.signature(generate_ti2ti)
_MAX_SEGS = 64  # sequences of one packed forward (kMaxSegs in csrc/mmdp_internal.h)


def batch_schedule(text_steps: Sequence[int], timesteps: Sequence[int]) -> List[tuple]:
    """The global steps of a batch: for global step g, (requests that run their step g, those of them in an image step).
    Request i runs its steps 0 .. text_steps[i] - 1 in order, its image steps at image_generation_step_indices."""
    img = [set(image_generation_step_indices(t, ts)) for t, ts in zip(text_steps, timesteps)]
    out = []
    for g in range(max(text_steps)):
        active = [i for i, t in enumerate(text_steps) if g < t]
        out.append((active, [i for i in active if g in img[i]]))
    return out


def packed_chunks(n_seqs: int, max_batch: int) -> List[range]:
    """Sequence index ranges of the packed forwards that serve n_seqs sequences, at most max_batch each."""
    return [range(i, min(i + max_batch, n_seqs)) for i in range(0, n_seqs, max_batch)]


def _bind(model, requests) -> List[dict]:
    """Every request's arguments with generate_ti2ti's defaults, checked before anything runs on the device."""
    if not requests:
        raise ValueError("generate_ti2ti_batch needs at least one request")
    args = []
    for r in requests:
        a = _SIGNATURE.bind(model, **r)
        a.apply_defaults()
        a = dict(a.arguments)
        check_request(model, a["input_ids"], a["remasking"])
        args.append(a)
    # a model with packed forwards exposes its capacity; an object without it (e.g. never constructed) is not a usable model
    if not hasattr(model, "forward_rows_packed") or not all(hasattr(model, k) for k in ("max_batch", "max_seq_len")):
        raise TypeError("generate_ti2ti_batch needs a constructed model with packed forwards and their capacity (max_batch, "
                        "max_seq_len): mmada_parallel_b200.model.LLaDAForMultiModalGeneration or "
                        "mmada_parallel_b200.tensor_parallel.TensorParallelLLaDA")
    seen = set()
    for i, a in enumerate(args):
        g = a["generator"]
        if not isinstance(g, torch.Generator):
            raise ValueError(f"request {i}: every request needs its own torch.Generator (got {g!r}); draws from a shared or "
                             "the global generator would interleave differently from sequential calls")
        if id(g) in seen:
            raise ValueError(f"request {i} shares its generator with an earlier request; each request needs its own")
        seen.add(id(g))
        L = a["input_ids"].shape[1]
        if L > model.max_seq_len:
            raise ValueError(f"request {i}: sequence of {L} tokens exceeds the model's max_seq_len={model.max_seq_len}")
        for key in ("uncon_text", "uncon_image"):
            u = a[key]
            if u is not None and u.shape[-1] > L:
                raise ValueError(f"request {i}: {key} has {u.shape[-1]} tokens, more than the sequence's {L}")
        for key in ("text_vocab_size", "codebook_size"):
            if a[key] != args[0][key]:
                raise ValueError(f"all requests of a batch share {key} (request {i}: {a[key]}, request 0: {args[0][key]})")
    return args


def _packed_forward(model, seqs: list, col0_b: int, ncols_b: int, windows=None) -> list:
    """Packed forwards over seqs = [(ids [L] cuda int64, text rows int32 or None, image rows int32 or None)], max_batch sequences
    per forward. windows (optional): the last-block row window (lo, hi) or None of every sequence. Returns [(text logits [n_a, V]
    or None, image logits [n_b, ncols_b] or None)] per sequence (views)."""
    outs = []
    for chunk in packed_chunks(len(seqs), min(model.max_batch, _MAX_SEGS)):
        part = [seqs[i] for i in chunk]
        lens = [s[0].numel() for s in part]
        offs = [sum(lens[:j]) for j in range(len(part))]
        ra = [s[1] + o for s, o in zip(part, offs) if s[1] is not None]
        rb = [s[2] + o for s, o in zip(part, offs) if s[2] is not None]
        win = None
        if windows is not None and any(windows[i] is not None for i in chunk):
            win = [windows[i] for i in chunk]
        out_a, out_b = model.forward_rows_packed(torch.cat([s[0] for s in part]), lens,
                                                 rows_a=torch.cat(ra) if ra else None, rows_b=torch.cat(rb) if rb else None,
                                                 col0_b=col0_b, ncols_b=ncols_b, row_windows=win)
        oa = ob = 0
        for s in part:
            va = vb = None
            if s[1] is not None:
                va, oa = out_a[oa:oa + s[1].numel()], oa + s[1].numel()
            if s[2] is not None:
                vb, ob = out_b[ob:ob + s[2].numel()], ob + s[2].numel()
            outs.append((va, vb))
    return outs


@torch.no_grad()
def generate_ti2ti_batch(model, requests: Sequence[dict]) -> list:
    """Runs the generate_ti2ti requests (dicts of its keyword arguments, without `model`) together and returns their results in
    request order: `[generate_ti2ti(model, **r) for r in requests]`. Each request needs its own torch.Generator. Argument
    errors raise before any forward; token ids outside the vocabulary raise IndexError after the loop."""
    args = _bind(model, requests)
    col0, ncols = args[0]["text_vocab_size"], args[0]["codebook_size"]
    states: List[DenoiseState] = []
    for a in args:
        states.append(DenoiseState(model, a["input_ids"].detach().to("cpu", torch.int64), a["text_start"], a["text_end"],
                                   a["image_start"], a["seq_len"], a["newline_every"], a["uncon_text"], a["uncon_image"],
                                   a["cfg_scale"], a["cfg_img"], a["codebook_size"]))
    num_transfer = [get_num_transfer_tokens(st.total_masks, a["text_steps"]) for st, a in zip(states, args)]
    noise = [_Noise(a["generator"], model.device) for a in args]
    masks_left = [st.total_masks for st in states]
    for g, (active, img) in enumerate(batch_schedule([a["text_steps"] for a in args], [a["timesteps"] for a in args])):
        img_set = set(img)
        # 1. conditional forward (:178) of every active request
        outs = _packed_forward(model, [(states[i].ids[0], states[i].text_rows, states[i].pos if i in img_set else None)
                                       for i in active], col0, ncols)
        # 2. text steps (:181-217)
        for i, (va, vb) in zip(active, outs):
            st, a = states[i], args[i]
            st.text_logits = va
            if vb is not None:
                st.cond_vq = vb
            text_sample(st, g, num_transfer[i][g], noise[i], a["text_temperature"], a["_trace"], masks_left[i])
            masks_left[i] -= num_transfer[i][g]
        # 3. unconditional forwards (:243-264) on the ids after the text steps
        seqs, targets = [], []
        for i in img:
            st, a = states[i], args[i]
            for name, prefix in uncond_inputs(st, a["cfg_scale"], a["cfg_img"]):
                x = st.ids[0].clone()
                if prefix is not None:
                    x[: prefix.shape[-1]] = prefix.reshape(-1)
                seqs.append((x, None, st.pos))
                targets.append((st, name))
        if seqs:
            for (st, name), (_, vb) in zip(targets, _packed_forward(model, seqs, col0, ncols)):
                setattr(st, name, vb)
        # 4. image steps (:220-344)
        for i in img:
            a = args[i]
            image_sample(states[i], g, noise[i], a["text_steps"], a["temperature"], a["cfg_scale"], a["cfg_img"],
                         a["noise_schedule"], a["text_vocab_size"], a["codebook_size"], a["_trace"])
    finals = [st.ids[0].cpu() for st in states]
    if hasattr(model, "raise_device_errors"):  # the tensor-parallel model has no device error flags (as in generate_ti2ti)
        model.raise_device_errors()
    results = []
    for st, a, final in zip(states, args, finals):
        image_tokens, text, _ = extract_results(st, final, a["tokenizer"], a["text_vocab_size"], a["codebook_size"])
        results.append((image_tokens, text))
    return results


def _bind_m(model, requests) -> List[dict]:
    """Every request's interleave_generate arguments with its defaults, checked before anything runs on the device."""
    from ..mmada import MMadaModelLM, interleave_layout
    if not requests:
        raise ValueError("interleave_generate_batch needs at least one request")
    sig = inspect.signature(MMadaModelLM.interleave_generate)
    args, seen = [], set()
    for i, r in enumerate(requests):
        a = sig.bind(model, **r)
        a.apply_defaults()
        a = dict(a.arguments)
        a.update(a.pop("kwargs"))
        if not (a["text_cfg"] or a["image_cfg"]):
            raise ValueError(f"request {i}: text_cfg and image_cfg cannot be both 0")
        if a["remasking"] != "low_confidence":
            raise NotImplementedError(a["remasking"])
        g = a["generator"]
        if not isinstance(g, torch.Generator):
            raise ValueError(f"request {i}: every request needs its own torch.Generator (got {g!r}); draws from a shared or "
                             "the global generator would interleave differently from sequential calls")
        if id(g) in seen:
            raise ValueError(f"request {i} shares its generator with an earlier request; each request needs its own")
        seen.add(id(g))
        if a["text_temperature"] != 0:
            raise ValueError(f"request {i}: text_temperature={a['text_temperature']} draws its Gumbel noise from the device's global "
                             "RNG, which sequential calls consume request after request; a batch cannot reproduce that order")
        lay = interleave_layout(a["config"], a.get("uni_prompting"), a["input_ids"], a["uncond_input_ids"], a["text_steps"],
                                a["image_steps"])
        if lay["L"] > model.max_seq_len:
            raise ValueError(f"request {i}: sequence of {lay['L']} tokens exceeds the model's max_seq_len={model.max_seq_len}")
        if not lay["img_idx"]:
            raise RuntimeError(f"request {i}: no image step was scheduled (the reference would hit an undefined `sampled_ids`)")
        for key, name in (("tvoc", "len(uni_prompting.text_tokenizer)"), ("C", "codebook_size")):
            if args and lay[key] != args[0]["_layout"][key]:
                raise ValueError(f"all requests of a batch share {name} (request {i}: {lay[key]}, request 0: {args[0]['_layout'][key]})")
        a["_layout"] = lay
        args.append(a)
    if not hasattr(model, "forward_rows_packed"):
        raise TypeError("interleave_generate_batch needs a model with packed forwards (mmada_parallel_b200.mmada.MMadaModelLM)")
    return args


@torch.no_grad()
def interleave_generate_batch(model, requests: Sequence[dict]) -> list:
    """Runs the variant-M interleave_generate requests (dicts of its keyword arguments) together and returns their results in
    request order: `[model.interleave_generate(**r) for r in requests]`, the (image_ids [1, num_vq_tokens], text_ids
    [1, max_seq_length]) tensors, with every request's generator left in the same state. Each request needs its own
    torch.Generator and text_temperature=0; all share the text vocabulary size and the codebook size. Argument errors raise
    before any forward."""
    from ..mmada import InterleaveState, interleave_image_step, interleave_text_step
    args = _bind_m(model, requests)
    col0, ncols = args[0]["_layout"]["tvoc"], args[0]["_layout"]["C"]
    states = [InterleaveState(model, **{k: v for k, v in a.items() if k not in ("self", "_layout")}) for a in args]
    steps = [a["text_steps"] for a in args]
    for g, (active, img) in enumerate(batch_schedule(steps, [a["image_steps"] for a in args])):
        img_set = set(img)
        # one packed forward (:172) over [cond; uncond] of every active request, each sequence with its own row window
        seqs, windows = [], []
        for i in active:
            st = states[i]
            rows_text = st.rows_text[:st.max_seq]
            for b in range(2):
                seqs.append((st.both[b], rows_text, st.pos if i in img_set else None))
                windows.append(st.window(g))
        outs = _packed_forward(model, seqs, col0, ncols, windows)
        for j, i in enumerate(active):
            (ta, ia), (tu, iu) = outs[2 * j], outs[2 * j + 1]
            interleave_text_step(states[i], g, ta, tu)
            if i in img_set:
                interleave_image_step(states[i], g, ia, iu)
    return [st.results() for st in states]
