"""Tensor-parallel grouped-query / multi-query attention and q/k/v-bias shards without a GPU: the kv-head sharding rule of
tensor_parallel.kv_shard / shard_state_dict on oracle.llada_gqa's weights, and the config checks of TensorParallelLLaDA's
constructor."""
import pytest
import torch

from oracle import llada_gqa

# (H, Hkv, tp): tp divides Hkv, Hkv divides tp (kv heads replicated; MQA), and multi-head shards
SHARD_CASES = [(8, 4, 2), (8, 2, 4), (8, 1, 4), (16, 4, 8), (16, 8, 2), (8, 8, 2), (8, 2, 1), (4, 1, 2)]


def _weights(H, Hkv, bias, n_layers=1):
    cfg = llada_gqa.make_config(d_model=H * 128, n_heads=H, n_kv_heads=Hkv, include_qkv_bias=bias, n_layers=n_layers,
                                mlp_hidden_size=1024, vocab_size=1024)
    return cfg, llada_gqa.make_weights(cfg, seed=H * 10 + (Hkv or 0))


def _shards(sd, cfg, tp, Hkv, bias):
    from mmada_parallel_b200.tensor_parallel import shard_state_dict
    return [shard_state_dict(sd, cfg.n_layers, cfg.n_heads, r, tp, 512, 256, n_kv_heads=Hkv, qkv_bias=bias) for r in range(tp)]


def _expected_kv_ranks(H, Hkv, tp, kv):
    """Ranks that must hold kv head `kv`: the ranks whose query heads read it."""
    Hl, G = H // tp, H // Hkv
    return sorted({h // Hl for h in range(H) if h // G == kv})


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("H,Hkv,tp", SHARD_CASES)
def test_q_rows_and_bias_concatenate(H, Hkv, tp, bias):
    cfg, sd = _weights(H, Hkv, bias)
    shards = _shards(sd, cfg, tp, Hkv, bias)
    p, da = "model.transformer.blocks.0.", (H // tp) * 128
    assert torch.equal(torch.cat([sh["blocks.0.wqkv"][:da] for sh in shards]), sd[p + "q_proj.weight"])
    if bias:
        assert torch.equal(torch.cat([sh["blocks.0.bqkv"][:da] for sh in shards]), sd[p + "q_proj.bias"])
    else:
        assert not any("bqkv" in k for sh in shards for k in sh)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("H,Hkv,tp", SHARD_CASES)
def test_kv_heads_on_exactly_the_ranks_that_read_them(H, Hkv, tp, bias):
    """Every kv head is on exactly the ranks whose query heads read it, with the full head's k and v rows (and bias), and local
    query head j of every rank reads (through the grouped attention's j // (Hl / Hkv_l)) the kv head its global head reads."""
    from mmada_parallel_b200.tensor_parallel import kv_shard
    cfg, sd = _weights(H, Hkv, bias)
    shards = _shards(sd, cfg, tp, Hkv, bias)
    p, Hl, G = "model.transformer.blocks.0.", H // tp, H // Hkv
    k_full, v_full = sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]
    held = {kv: [] for kv in range(Hkv)}
    for r, sh in enumerate(shards):
        kv0, n_kv = kv_shard(H, Hkv, r, tp)
        assert n_kv == (Hkv // tp if Hkv % tp == 0 else 1)
        w = sh["blocks.0.wqkv"]
        assert w.shape == ((Hl + 2 * n_kv) * 128, cfg.d_model)
        k_loc, v_loc = w[Hl * 128:(Hl + n_kv) * 128], w[(Hl + n_kv) * 128:]
        for j in range(n_kv):
            kv = kv0 + j
            rows = slice(kv * 128, (kv + 1) * 128)
            assert torch.equal(k_loc[j * 128:(j + 1) * 128], k_full[rows]) and torch.equal(v_loc[j * 128:(j + 1) * 128], v_full[rows])
            if bias:
                b = sh["blocks.0.bqkv"]
                assert b.shape == ((Hl + 2 * n_kv) * 128,)
                assert torch.equal(b[(Hl + j) * 128:(Hl + j + 1) * 128], sd[p + "k_proj.bias"][rows])
                assert torch.equal(b[(Hl + n_kv + j) * 128:(Hl + n_kv + j + 1) * 128], sd[p + "v_proj.bias"][rows])
            held[kv].append(r)
        for j in range(Hl):
            assert kv0 + j // (Hl // n_kv) == (r * Hl + j) // G, f"rank {r} local head {j} reads the wrong kv head"
    for kv in range(Hkv):
        assert held[kv] == _expected_kv_ranks(H, Hkv, tp, kv), (kv, held[kv])


@pytest.mark.parametrize("H,tp", [(4, 1), (4, 2), (8, 4), (16, 8)])
def test_multi_head_shards_unchanged(H, tp):
    """A multi-head config without a bias: the same keys and tensors as the head split of the multi-head layout (q | k | v rows
    of the local heads), whether n_kv_heads is left out, None or n_heads."""
    from mmada_parallel_b200.tensor_parallel import shard_state_dict
    cfg, sd = _weights(H, None, False, n_layers=2)
    da = (H // tp) * 128
    for r in range(tp):
        base = shard_state_dict(sd, cfg.n_layers, H, r, tp, 512, 256)
        sl = slice(r * da, (r + 1) * da)
        for i in range(cfg.n_layers):
            p = f"model.transformer.blocks.{i}."
            want = torch.cat([sd[p + "q_proj.weight"][sl], sd[p + "k_proj.weight"][sl], sd[p + "v_proj.weight"][sl]])
            assert torch.equal(base[f"blocks.{i}.wqkv"], want)
        for kw in (dict(n_kv_heads=None), dict(n_kv_heads=H), dict(n_kv_heads=H, qkv_bias=False)):
            other = shard_state_dict(sd, cfg.n_layers, H, r, tp, 512, 256, **kw)
            assert other.keys() == base.keys() and all(torch.equal(other[k], base[k]) for k in base)


@pytest.mark.parametrize("H,Hkv,tp", [(12, 3, 2), (24, 6, 4), (20, 5, 2)])
def test_incompatible_tp_and_kv_heads_raise(H, Hkv, tp):
    """Neither of tp and Hkv divides the other: one rank's query heads would read kv heads of two ranks."""
    from mmada_parallel_b200.tensor_parallel import shard_state_dict
    cfg, sd = _weights(H, Hkv, False)
    with pytest.raises(ValueError, match=rf"tp={tp} and n_kv_heads={Hkv}"):
        shard_state_dict(sd, 1, H, 0, tp, 512, 256, n_kv_heads=Hkv)
    with pytest.raises(ValueError, match=rf"tp={tp} and n_kv_heads={Hkv}"):
        _tp_model(cfg, sd, 0, tp)


def _tp_model(cfg, sd, rank, tp):
    """TensorParallelLLaDA's constructor on the CPU: with tp_size 1 or the NCCL collective it needs no peer buffers and no
    process group, and its weights and work buffers may live on any torch device. Only the device check is bypassed."""
    from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA
    mp = pytest.MonkeyPatch()
    mp.setattr(torch.cuda, "is_available", lambda: True)
    mp.setattr(torch.cuda, "set_device", lambda *_: None)
    try:
        return TensorParallelLLaDA(cfg, sd, rank, tp, max_seq_len=64, device="cpu", text_vocab_size=512, codebook_size=256,
                                   collective="nccl")
    finally:
        mp.undo()


@pytest.mark.parametrize("kw,tp,kv_local", [(dict(n_kv_heads=2, include_qkv_bias=True), 2, 1), (dict(multi_query_attention=True), 4, 1),
                                            (dict(n_kv_heads=8, include_qkv_bias=True), 2, 4), (dict(n_kv_heads=4), 8, 1)])
def test_tp_model_accepts_grouped_query_and_bias(kw, tp, kv_local):
    cfg = llada_gqa.make_config(d_model=2048, n_heads=16, n_layers=1, mlp_hidden_size=1024, vocab_size=1024, **kw)
    sd = llada_gqa.make_weights(cfg, seed=1)
    for rank in (0, tp - 1):
        m = _tp_model(cfg, sd, rank, tp)
        assert (m.n_kv_heads, m.kv_local, m.qkv_bias, m.gqa) == (llada_gqa.kv_heads(cfg), kv_local, bool(cfg.include_qkv_bias), True)
        assert m.k.shape == (64, 128 * kv_local) and m.q.shape == (64, 128 * (16 // tp))
        assert ("blocks.0.bqkv" in m.w) == bool(cfg.include_qkv_bias)
    cfg = llada_gqa.make_config(d_model=2048, n_heads=16, n_layers=1, mlp_hidden_size=1024, vocab_size=1024)
    plain = _tp_model(cfg, llada_gqa.make_weights(cfg, seed=1), 0, 2)
    assert not plain.gqa and plain.kv_local == plain.h_local == 8 and "blocks.0.bqkv" not in plain.w


@pytest.mark.parametrize("flag", ["include_bias", "alibi", "attention_layer_norm", "weight_tying", "scale_logits", "input_emb_norm"])
def test_tp_model_still_refuses_other_flags(flag):
    cfg = llada_gqa.make_config(d_model=512, n_heads=4, n_layers=1, mlp_hidden_size=1024, vocab_size=1024, n_kv_heads=2,
                                include_qkv_bias=True)
    setattr(cfg, flag, True)
    with pytest.raises(NotImplementedError, match=flag):
        _tp_model(cfg, llada_gqa.make_weights(cfg, seed=2), 0, 2)
