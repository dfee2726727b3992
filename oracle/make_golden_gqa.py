"""Writes tests/golden/forward_gqa_tiny.pt: grouped-query / multi-query attention and q/k/v-bias configs of the REAL reference
(LLaDALlamaBlock with effective_n_kv_heads < n_heads and include_qkv_bias, modeling_llada.py:660-679, :866-884), pinning the
oracle (oracle.llada_gqa) to it bit for bit.

    MMDP_REFERENCE_ROOT=<checkout> PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_gqa

Three configs: H=4 with n_kv_heads=2 and a q/k/v bias, H=4 with multi_query_attention=True (one kv head) and H=2 with
n_kv_heads=2 and a bias. The reference initialises the biases to zero; the recipe loads seeded non-zero ones
(oracle.llada_gqa.make_weights). Per config: logits at B=1 and B=2 (a subset of columns) and one greedy generate_ti2ti trajectory.
"""
from __future__ import annotations

import os

import torch

from . import generate as G
from . import llada_gqa
from . import ref_shim
from .make_golden import OUT, layout_a, quiet

CONFIGS = {
    "h4_kv2_bias": dict(d_model=512, n_heads=4, n_kv_heads=2, include_qkv_bias=True),
    "h4_mqa": dict(d_model=512, n_heads=4, multi_query_attention=True),
    "h2_kv2_bias": dict(d_model=256, n_heads=2, n_kv_heads=2, include_qkv_bias=True),
}
COMMON = dict(n_layers=2, mlp_hidden_size=512, vocab_size=134656, max_sequence_length=512)
WEIGHT_SEED = 4321
GREEDY = dict(temperature=0.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0, text_steps=8, text_gen_length=16,
              text_block_length=4, timesteps=4, tokenizer=None, text_vocab_size=126356, codebook_size=8192)


def build_ref(cfg, sd):
    Model, _, _, _ = ref_shim.load_a()
    rc = ref_shim.ref_config_a(cfg)
    rc.n_kv_heads = cfg.n_kv_heads
    rc.multi_query_attention = cfg.multi_query_attention
    rc.include_qkv_bias = cfg.include_qkv_bias
    m = Model(rc, init_params=False).eval().to(torch.bfloat16)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in k or "inv_freq" in k for k in missing), missing
    blk = m.model.transformer.blocks[0]
    assert blk.k_proj.weight.shape[0] == llada_gqa.kv_heads(cfg) * 128
    assert (blk.q_proj.bias is not None) == cfg.include_qkv_bias
    return m


def main():
    assert ref_shim.available(), "reference tree not found"
    torch.set_num_threads(8)
    _, _, pg, _ = ref_shim.load_a()
    lay = layout_a()
    ids = lay["input_ids"]
    ids2 = torch.cat([ids, ids.flip(1)], dim=0)
    cols = torch.cat([torch.arange(0, 134656, 997), torch.arange(126356, 126356 + 8192, 61)])
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    out = dict(meta=dict(common=COMMON, weight_seed=WEIGHT_SEED, greedy=GREEDY), layout=lay, ids=ids, ids2=ids2, cols=cols,
               configs={})
    for name, kw in CONFIGS.items():
        cfg = llada_gqa.make_config(**COMMON, **kw)
        sd = llada_gqa.make_weights(cfg, seed=WEIGHT_SEED)
        with quiet():
            ref = build_ref(cfg, sd)
        oracle_model = llada_gqa.OracleModel(cfg, sd)
        with torch.no_grad():
            lr = ref(ids, infer=True, use_cache=False).logits
            lr2 = ref(ids2, infer=True, use_cache=False).logits
        assert torch.equal(lr, oracle_model(ids).logits), f"{name}: oracle forward != reference forward"
        assert torch.equal(lr2, oracle_model(ids2).logits), f"{name}: oracle B=2 forward != reference forward"
        torch.manual_seed(999)
        with quiet():
            img_r, txt_r = pg.generate_ti2ti(ref, ids, generator=torch.Generator().manual_seed(42), **args, **GREEDY)
        torch.manual_seed(999)
        img_o, txt_o = G.generate_ti2ti(oracle_model, ids, generator=torch.Generator().manual_seed(42), **args, **GREEDY)
        assert img_r == img_o and txt_r == txt_o, f"{name}: oracle trajectory != reference trajectory"
        out["configs"][name] = dict(config=kw, logits_cols=lr[0][:, cols].clone(), logits2_cols=lr2[:, :, cols].clone(),
                                    argmax=lr[0].argmax(-1), image_tokens=img_r, text_tokens=txt_r)
        print(name, "ok", tuple(lr.shape), "kv heads", llada_gqa.kv_heads(cfg), "text tokens", len(txt_r))
    torch.save(out, os.path.join(OUT, "forward_gqa_tiny.pt"))
    print("forward_gqa_tiny.pt written to", OUT)


if __name__ == "__main__":
    main()
