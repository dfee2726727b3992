"""Grouped-query / multi-query attention and q/k/v-bias configs without a GPU: the oracle against the real reference's fixture
(tests/golden/forward_gqa_tiny.pt, oracle/make_golden_gqa.py) bit for bit, and the config and ABI checks that run before any
device work."""
import ctypes as C
import functools

import pytest
import torch

from helpers import load_golden
from oracle import generate as G
from oracle import llada, llada_gqa


def _gqa_cfg(g, name):
    return llada_gqa.make_config(**g["meta"]["common"], **g["configs"][name]["config"])


@functools.lru_cache(maxsize=1)
def host_rounds_like_fixtures() -> bool:
    """Whether this host's torch-CPU bf16 kernels reproduce the multi-head fixture (forward_tiny.pt) bit for bit. The fixtures
    were recorded on a CPU whose bf16 matmuls round like the reference run's; a CPU with other bf16 kernels (another vector
    ISA) rounds some products differently, and then no oracle can match any fixture bit for bit."""
    g = load_golden("forward_tiny.pt")
    cfg = llada.make_config(**g["meta"]["tiny"])
    lg = llada.OracleModel(cfg, llada.make_weights(cfg, seed=g["meta"]["weight_seed"]))(g["ids"]).logits
    return torch.equal(lg[0][:, g["cols"]], g["logits_cols"])


@pytest.mark.parametrize("name", ["h4_kv2_bias", "h4_mqa", "h2_kv2_bias"])
def test_oracle_matches_reference_gqa_golden(name):
    """Bit for bit (logits at B=1 and B=2, the greedy trajectory) where the host reproduces the multi-head fixture bit for bit;
    elsewhere the logits within 4 bf16 ulp of their scale."""
    g = load_golden("forward_gqa_tiny.pt")
    c = g["configs"][name]
    cfg = _gqa_cfg(g, name)
    sd = llada_gqa.make_weights(cfg, seed=g["meta"]["weight_seed"])
    model = llada_gqa.OracleModel(cfg, sd)
    lg = model(g["ids"]).logits
    lg2 = model(g["ids2"]).logits
    if not host_rounds_like_fixtures():
        tol = 4 * c["logits_cols"].float().abs().max().item() * 2.0 ** -8
        assert (lg[0][:, g["cols"]].float() - c["logits_cols"].float()).abs().max().item() <= tol
        assert (lg2[:, :, g["cols"]].float() - c["logits2_cols"].float()).abs().max().item() <= tol
        pytest.skip("this host's CPU bf16 kernels do not reproduce the multi-head fixture bit for bit: logits checked to 4 ulp only")
    assert torch.equal(lg[0][:, g["cols"]], c["logits_cols"])
    assert torch.equal(lg[0].argmax(-1), c["argmax"])
    assert torch.equal(lg2[:, :, g["cols"]], c["logits2_cols"])
    lay = g["layout"]
    args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
    torch.manual_seed(999)
    img, txt = G.generate_ti2ti(model, g["ids"], generator=torch.Generator().manual_seed(42), **args, **g["meta"]["greedy"])
    assert img == c["image_tokens"] and txt == c["text_tokens"]


def test_gqa_oracle_is_the_multi_head_oracle_without_kv_groups_or_bias():
    """oracle.llada_gqa with n_kv_heads == n_heads and no bias: oracle.llada's weights and logits, bit for bit."""
    cfg = llada.make_config(d_model=256, n_heads=2, vocab_size=1024)
    sd = llada.make_weights(cfg, seed=5)
    sd_g = llada_gqa.make_weights(llada_gqa.make_config(d_model=256, n_heads=2, vocab_size=1024), seed=5)
    assert sd.keys() == sd_g.keys() and all(torch.equal(v, sd_g[k]) for k, v in sd.items())
    ids = torch.randint(0, 1024, (2, 37), generator=torch.Generator().manual_seed(1))
    assert torch.equal(llada_gqa.OracleModel(cfg, sd)(ids).logits, llada.OracleModel(cfg, sd)(ids).logits)
    from oracle import fp8, fp8_gqa
    assert torch.equal(fp8_gqa.forward_logits_fp8(ids, sd, cfg), fp8.forward_logits_fp8(ids, sd, cfg))


def test_gqa_weights_shapes_and_bias_draws():
    cfg = llada_gqa.make_config(d_model=512, n_heads=4, n_kv_heads=2, include_qkv_bias=True, vocab_size=1024)
    sd = llada_gqa.make_weights(cfg, seed=3)
    p = "model.transformer.blocks.0."
    assert sd[p + "k_proj.weight"].shape == (256, 512) and sd[p + "v_proj.bias"].shape == (256,)
    assert sd[p + "q_proj.bias"].shape == (512,) and sd[p + "q_proj.bias"].abs().max() > 0
    # the bias is drawn last: every other tensor equals that of the config without a bias
    plain = llada_gqa.make_weights(llada_gqa.make_config(d_model=512, n_heads=4, n_kv_heads=2, vocab_size=1024), seed=3)
    assert all(torch.equal(v, sd[k]) for k, v in plain.items()) and len(sd) == len(plain) + 6


def test_effective_kv_heads_and_refusals():
    from mmada_parallel_b200.model import check_supported_config, effective_n_kv_heads

    def cfg(**kw):
        return llada_gqa.make_config(d_model=512, n_heads=4, **kw)

    assert effective_n_kv_heads(cfg(), 4) == 4
    assert effective_n_kv_heads(cfg(n_kv_heads=2), 4) == 2
    assert effective_n_kv_heads(cfg(multi_query_attention=True), 4) == 1  # MQA by flag: one kv head
    assert effective_n_kv_heads(cfg(n_kv_heads=1, multi_query_attention=True), 4) == 1
    assert effective_n_kv_heads(cfg(n_kv_heads=4, multi_query_attention=False), 4) == 4
    with pytest.raises(ValueError, match="at the same time"):
        effective_n_kv_heads(cfg(n_kv_heads=2, multi_query_attention=True), 4)
    with pytest.raises(ValueError, match="divide"):
        effective_n_kv_heads(cfg(n_kv_heads=3), 4)
    # the single-GPU model runs grouped-query and q/k/v-bias configs, the tensor-parallel model refuses them
    assert check_supported_config(cfg(multi_query_attention=True, include_qkv_bias=True), 4, grouped_query=True) == 1
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        check_supported_config(cfg(multi_query_attention=True), 4)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        check_supported_config(cfg(include_qkv_bias=True), 4)
    with pytest.raises(ValueError):
        check_supported_config(cfg(n_kv_heads=3), 4, grouped_query=True)
    for flag in ("include_bias", "alibi", "attention_layer_norm", "weight_tying", "scale_logits", "input_emb_norm"):
        c = cfg(n_kv_heads=2)
        setattr(c, flag, True)
        with pytest.raises(NotImplementedError, match=flag):
            check_supported_config(c, 4, grouped_query=True)


def test_create_arch_validates_before_device_work():
    from mmada_parallel_b200 import _lib
    cfg = _lib.ModelConfig(512, 4, 2, 512, 134656, 512, 2, 1e-5)
    h = C.c_void_p()
    assert _lib.lib.mmdp_model_create_arch(C.byref(cfg), 0, 3, 0, C.byref(h)) == -1
    assert b"n_kv_heads=3 must divide n_heads=4" in _lib.lib.mmdp_last_error()
    assert _lib.lib.mmdp_model_create_arch(C.byref(cfg), 0, 8, 0, C.byref(h)) == -1
    assert _lib.lib.mmdp_model_create_arch(C.byref(cfg), 0, 2, 6, C.byref(h)) == -1
    assert b"flags" in _lib.lib.mmdp_last_error()
    if not torch.cuda.is_available():
        assert _lib.lib.mmdp_model_create_arch(C.byref(cfg), 0, 1, _lib.ARCH_QKV_BIAS, C.byref(h)) == -1
        assert b"no CUDA device" in _lib.lib.mmdp_last_error()


def test_bias_weight_names():
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration as M
    f = M._native_name
    assert f("model.transformer.blocks.3.k_proj.bias", True) == "blocks.3.k_bias"
    assert f("model.transformer.blocks.3.q_proj.bias", True) == "blocks.3.q_bias"
    assert f("model.transformer.blocks.3.k_proj.bias") is None  # not a tensor of a context without the bias
    assert f("model.transformer.blocks.3.ff_proj.bias", True) is None
    cfg = llada_gqa.make_config(d_model=256, n_heads=2, n_kv_heads=2, include_qkv_bias=True, vocab_size=1024)
    names = {f(k, True) for k in llada_gqa.make_weights(cfg, 0)}
    assert None not in names and len(names) == 3 + 12 * cfg.n_layers
