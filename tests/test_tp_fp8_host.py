"""The FP8 tensor-parallel contract without a GPU (DESIGN §3 "FP8 under tensor parallel"):

  oracle.fp8_tp at tp = 1          bit for bit oracle.fp8_gqa's block (multi-head, kv heads + bias, MQA)
  oracle.fp8_tp at tp = 2 / 4      only the fp32 summation order of attn_out / ff_out moves: close to tp = 1
  activation groups                a rank's K-slice of the quantised att / h is the quantisation of its slice (whole groups)
  shard_state_dict_fp8             every byte and scale a rank holds is a slice of the single-GPU quantisation: the rows of its
                                   heads / kv heads (including the replicated multi-query kv head) / ff columns, the K-columns
                                   of attn_out and ff_out with their full row scales, W13 in 64-row gate / up blocks
  TensorParallelLLaDA(precision)   anything but "bf16" / "fp8" is a ValueError"""
import pytest
import torch

from oracle import fp8, fp8_gqa, fp8_tp, llada, llada_gqa

CONFIGS = {"mha": dict(), "kv2_bias": dict(n_kv_heads=2, include_qkv_bias=True), "mqa": dict(multi_query_attention=True)}


def _model(name, H=4, n_layers=1, ff=1024, seed=5):
    cfg = llada_gqa.make_config(d_model=H * 128, n_heads=H, n_layers=n_layers, mlp_hidden_size=ff, vocab_size=256, **CONFIGS[name])
    return cfg, llada_gqa.make_weights(cfg, seed=seed)


def _block(cfg, w, wq, x, tp):
    pos_sin, pos_cos = llada.rotary_tables(128, cfg.rope_theta, x.shape[1])
    p = "model.transformer.blocks.0."
    if tp is None:
        return fp8_gqa.block_forward_fp8(x, w, wq, p, cfg, pos_sin, pos_cos)
    return fp8_tp.block_forward_tp_fp8(x, w, wq, p, cfg, pos_sin, pos_cos, tp)


def _x(cfg, B=2, T=24, seed=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, T, cfg.d_model, generator=g)).to(torch.bfloat16)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_tp1_oracle_is_the_single_gpu_fp8_block(name):
    cfg, w = _model(name)
    wq = fp8.quantize_weights(w)
    x = _x(cfg)
    assert torch.equal(_block(cfg, w, wq, x, 1), _block(cfg, w, wq, x, None))


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("tp", [2, 4])
def test_tp_oracle_differs_only_by_the_partial_sum_order(name, tp):
    """attn_out / ff_out summed over tp fp32 partials: every element within a few bf16 ulp of the tensor's scale of tp = 1."""
    cfg, w = _model(name)
    wq = fp8.quantize_weights(w)
    x = _x(cfg, seed=tp)
    one, many = _block(cfg, w, wq, x, 1).float(), _block(cfg, w, wq, x, tp).float()
    ulp = one.abs().max().item() * 2.0 ** -8
    err = (many - one).abs()
    assert err.max().item() <= 4 * ulp, err.max().item() / ulp
    assert err.mean().item() <= 0.05 * ulp, err.mean().item() / ulp


@pytest.mark.parametrize("tp", [2, 4, 8])
def test_rank_slices_hold_whole_activation_groups(tp):
    g = torch.Generator().manual_seed(tp)
    K = 1024
    a = (torch.randn(37, K, generator=g) * torch.logspace(-3, 2, K).unsqueeze(0)).to(torch.bfloat16)
    q, s = fp8.quantize_fp8(a, fp8.ACT_GROUP)
    k, ng = K // tp, K // tp // 128
    for r in range(tp):
        qr, sr = fp8.quantize_fp8(a[:, r * k:(r + 1) * k].contiguous(), fp8.ACT_GROUP)
        assert torch.equal(qr.view(torch.uint8), q[:, r * k:(r + 1) * k].view(torch.uint8))
        assert torch.equal(sr, s[r * ng:(r + 1) * ng])


def _oracle_quantize(w):
    q, s = fp8.quantize_fp8(w, w.shape[1])
    return q.view(torch.uint8), s[0]


# (H, Hkv, tp): multi-head, tp divides Hkv, Hkv divides tp (replicated kv heads), MQA replicated on every rank
SHARD_CASES = [(4, 4, 2), (8, 4, 2), (8, 2, 4), (8, 1, 4), (4, 2, 1), (8, 4, 8)]


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("H,Hkv,tp", SHARD_CASES)
def test_fp8_shards_are_slices_of_the_full_quantisation(H, Hkv, tp, bias):
    from mmada_parallel_b200.tensor_parallel import shard_state_dict, shard_state_dict_fp8
    cfg = llada_gqa.make_config(d_model=H * 128, n_heads=H, n_kv_heads=Hkv, include_qkv_bias=bias, n_layers=2, mlp_hidden_size=128 * tp * 2,
                                vocab_size=256)
    sd = llada_gqa.make_weights(cfg, seed=H + Hkv + tp)
    wq = {k: (q.view(torch.uint8), s) for k, (q, s) in fp8.quantize_weights(sd).items()}
    d, ff, Hl = cfg.d_model, cfg.mlp_hidden_size, H // tp
    for r in range(tp):
        sh = shard_state_dict_fp8(sd, cfg.n_layers, H, r, tp, _oracle_quantize, n_kv_heads=Hkv)
        ref = fp8_tp.shard_fp8(wq, cfg, r, tp)
        bf = shard_state_dict(sd, cfg.n_layers, H, r, tp, 0, 256, n_kv_heads=Hkv, qkv_bias=bias)
        for i in range(cfg.n_layers):
            p, P = f"blocks.{i}.", f"model.transformer.blocks.{i}."
            # q rows of the rank's heads, k / v rows of its kv heads: the rows of the bf16 shard, quantised as the full weight
            want_q = torch.cat([ref[P + n + ".weight"][0] for n in ("q_proj", "k_proj", "v_proj")])
            want_s = torch.cat([ref[P + n + ".weight"][1] for n in ("q_proj", "k_proj", "v_proj")])
            assert sh[p + "wqkv8"].dtype == torch.uint8 and sh[p + "wqkv8"].shape == bf[p + "wqkv"].shape
            assert torch.equal(sh[p + "wqkv8"], want_q) and torch.equal(sh[p + "sqkv"], want_s)
            # row-parallel: K-columns of the bytes, the FULL row scales
            assert sh[p + "wo8"].shape == (d, Hl * 128) and torch.equal(sh[p + "wo8"], wq[P + "attn_out.weight"][0][:, r * Hl * 128:(r + 1) * Hl * 128])
            assert torch.equal(sh[p + "so"], wq[P + "attn_out.weight"][1]) and sh[p + "so"].shape == (d,)
            f = ff // tp
            assert torch.equal(sh[p + "w2_8"], wq[P + "ff_out.weight"][0][:, r * f:(r + 1) * f])
            assert torch.equal(sh[p + "s2"], wq[P + "ff_out.weight"][1])
            # W13: block 2t = gate rows [64t, 64t + 64) of the shard, block 2t + 1 = the same up rows
            (g8, gs), (u8, us) = ref[P + "ff_proj.weight"], ref[P + "up_proj.weight"]
            w13, s13 = sh[p + "w13_8"].view(f // 64, 2, 64, d), sh[p + "s13"].view(f // 64, 2, 64)
            assert torch.equal(w13[:, 0].reshape(f, d), g8) and torch.equal(w13[:, 1].reshape(f, d), u8)
            assert torch.equal(s13[:, 0].reshape(f), gs) and torch.equal(s13[:, 1].reshape(f), us)


def test_mqa_kv_head_replicated_on_every_rank():
    from mmada_parallel_b200.tensor_parallel import shard_state_dict_fp8
    cfg = llada_gqa.make_config(d_model=1024, n_heads=8, multi_query_attention=True, n_layers=1, mlp_hidden_size=1024, vocab_size=256)
    sd = llada_gqa.make_weights(cfg, seed=11)
    kq, ks = _oracle_quantize(sd["model.transformer.blocks.0.k_proj.weight"])
    for r in range(4):
        sh = shard_state_dict_fp8(sd, 1, 8, r, 4, _oracle_quantize, n_kv_heads=1)
        assert torch.equal(sh["blocks.0.wqkv8"][256:384], kq) and torch.equal(sh["blocks.0.sqkv"][256:384], ks)


def test_tp1_shard_is_the_single_gpu_fp8_weights():
    """At tp = 1 the shard is the FP8 context's packed weights: q | k | v rows, and W13 interleaved in 64-row blocks as
    mmdp_model_set_weight packs it (source block t -> destination block 2t + up)."""
    from mmada_parallel_b200.tensor_parallel import shard_state_dict_fp8
    cfg, sd = _model("kv2_bias")
    sh = shard_state_dict_fp8(sd, 1, cfg.n_heads, 0, 1, _oracle_quantize, n_kv_heads=2)
    P = "model.transformer.blocks.0."
    g8, _ = _oracle_quantize(sd[P + "ff_proj.weight"])
    u8, _ = _oracle_quantize(sd[P + "up_proj.weight"])
    ff, d = g8.shape
    packed = torch.empty(2 * ff, d, dtype=torch.uint8)
    for t in range(ff // 64):
        packed[128 * t:128 * t + 64] = g8[64 * t:64 * t + 64]
        packed[128 * t + 64:128 * t + 128] = u8[64 * t:64 * t + 64]
    assert torch.equal(sh["blocks.0.w13_8"], packed)
    assert torch.equal(sh["blocks.0.wo8"], _oracle_quantize(sd[P + "attn_out.weight"])[0])


def test_precision_argument_is_checked():
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    for bad in ("fp16", "FP8", None):
        with pytest.raises(ValueError, match="precision"):
            TensorParallelLLaDA(None, {}, 0, 1, precision=bad)
