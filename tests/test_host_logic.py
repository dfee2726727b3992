"""Host-side logic of the product package (no GPU): schedules, weight-name mapping, replica sharding (gloo, world 2)."""
import os
import socket
import subprocess
import sys

import torch

from helpers import ROOT
from oracle import sampling as S


def test_schedules_match_oracle():
    from mmada_parallel_b200 import schedule as P
    for n, steps in [(256, 128), (16, 8), (100, 7), (5, 9), (0, 4), (1, 1)]:
        assert P.get_num_transfer_tokens(n, steps) == S.get_num_transfer_tokens_a(n, steps)
        assert P.get_num_transfer_tokens_m(n, steps) == S.get_num_transfer_tokens_m(n, steps)
    for ts, t in [(128, 64), (8, 4), (100, 100), (128, 128), (50, 30)]:
        assert P.image_generation_step_indices(ts, t) == S.image_step_indices(ts, t)
    assert [P.scheduled_mask_len(1024, s, 128) for s in range(128)] == [S.sched_len(1024, s, 128) for s in range(128)]
    assert P.scheduled_mask_len(1024, 127, 128) == -1
    m = torch.zeros(2, 10, dtype=torch.bool)
    m[0, :7] = True
    from mmada_parallel_b200.generators.parallel_generator import get_num_transfer_tokens
    out = get_num_transfer_tokens(m, 4)
    assert out.shape == (2, 4) and out[0].tolist() == S.get_num_transfer_tokens_a(7, 4) and out[1].tolist() == [0, 0, 0, 0]


def test_weight_name_mapping():
    from mmada_parallel_b200.model import LLaDAForMultiModalGeneration as M
    f = M._native_name
    assert f("model.transformer.wte.weight") == "wte"
    assert f("model.transformer.ff_out.weight") == "head"
    assert f("model.transformer.ln_f.weight") == "ln_f"
    assert f("model.transformer.blocks.17.ff_out.weight") == "blocks.17.ff_out"
    assert f("model.transformer.blocks.0.up_proj.weight") == "blocks.0.up_proj"
    assert f("model.transformer.blocks.0.rotary_emb.inv_freq") is None
    from oracle.llada import make_config, make_weights
    cfg = make_config(vocab_size=1024, d_model=256)
    names = {f(k) for k in make_weights(cfg, 0)}
    assert None not in names and len(names) == 3 + 9 * cfg.n_layers


def test_rope_table_matches_reference_formula():
    from mmada_parallel_b200.model import rope_tables
    from oracle.llada import rotary_tables
    cos, sin = rope_tables(128, 500000.0, 300)
    s, c = rotary_tables(128, 500000.0, 300)
    assert torch.equal(cos, c[0, 0, :, :64]) and torch.equal(cos, c[0, 0, :, 64:])
    assert torch.equal(sin, s[0, 0, :, :64]) and torch.equal(sin, s[0, 0, :, 64:])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_replica_sharding_gloo_world2():
    """bench.py's multi-GPU mode = independent prompt replicas + a max-over-ranks time reduction; exercised here with
    gloo on CPU (world_size 2): disjoint prompt shards that cover the job, and the reduction returns the slowest rank."""
    port = _free_port()
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_gloo_worker.py")],
                              env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for r in range(2)]
    outs = [p.communicate(timeout=180) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, e[-2000:]
    assert "OK rank0 shard=[0, 2, 4] max_ms=20.0 total=5" in outs[0][0]
    assert "OK rank1 shard=[1, 3] max_ms=20.0 total=5" in outs[1][0]


def test_tensor_parallel_sharding_math():
    """shard_state_dict: per-rank shards reproduce the full projections (column-parallel outputs concatenate,
    row-parallel partial products sum) - checked in fp64 on the CPU."""
    from mmada_parallel_b200.tensor_parallel import shard_state_dict
    from oracle.llada import make_config, make_weights
    cfg = make_config(d_model=512, n_heads=4, n_layers=1, mlp_hidden_size=1024, vocab_size=1024)
    sd = {k: v.double() for k, v in make_weights(cfg, 3).items()}
    tp, d = 2, cfg.d_model
    shards = [shard_state_dict(sd, 1, cfg.n_heads, r, tp, vq_col0=512, vq_cols=256) for r in range(tp)]
    x = torch.randn(7, d, dtype=torch.float64)
    p = "model.transformer.blocks.0."
    q_full = x @ sd[p + "q_proj.weight"].t()
    da = d // tp
    q_cat = torch.cat([x @ sh["blocks.0.wqkv"][:da].t() for sh in shards], dim=1)
    v_cat = torch.cat([x @ sh["blocks.0.wqkv"][2 * da:].t() for sh in shards], dim=1)
    assert torch.allclose(q_cat, q_full) and torch.allclose(v_cat, x @ sd[p + "v_proj.weight"].t())
    att = torch.randn(7, d, dtype=torch.float64)
    part = sum(att[:, r * da:(r + 1) * da] @ shards[r]["blocks.0.wo"].t() for r in range(tp))
    assert torch.allclose(part, att @ sd[p + "attn_out.weight"].t())
    # SwiGLU shard: interleaved 128-row gate/up blocks, then the row-parallel ff_out partials sum to the full MLP
    def mlp_local(sh):
        w13 = sh["blocks.0.w13"].reshape(-1, 2, 128, d)
        g, u = x @ w13[:, 0].reshape(-1, d).t(), x @ w13[:, 1].reshape(-1, d).t()
        return (torch.nn.functional.silu(g) * u) @ sh["blocks.0.w2"].t()
    full = (torch.nn.functional.silu(x @ sd[p + "ff_proj.weight"].t()) * (x @ sd[p + "up_proj.weight"].t())) @ sd[p + "ff_out.weight"].t()
    assert torch.allclose(sum(mlp_local(sh) for sh in shards), full)
    head = sd["model.transformer.ff_out.weight"]
    assert torch.equal(torch.cat([sh["head"] for sh in shards]), head)
    assert torch.equal(torch.cat([sh["head_vq"] for sh in shards]), head[512:768])


def test_gemm_tile_order_is_a_bijection(tmp_path):
    """The grouped-M tile order of the persistent GEMM (csrc/gemm_epilogue.cuh::gemm_tile_coords) visits every tile exactly
    once for every group size, and halves the m-span of a 132-tile wave at 57 m-tiles. Host-only: the function is
    __host__ __device__, the check is compiled with nvcc and runs on the CPU (tests/host/tile_order.cu)."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "tile_order")
    subprocess.run([nvcc, "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host", "tile_order.cu")], check=True,
                   capture_output=True, timeout=300)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr


def test_preview_host_helpers_match_oracle():
    """Host-side pieces of the step-wise preview path (no GPU work): text rendering and image-step schedule equal the pinned
    oracle; decode_vq_to_image's conversion / overlay / error contract with a stand-in decoder (A/utils/image_utils.py:13-75,
    A/app.py:312-333)."""
    from types import SimpleNamespace
    from oracle import generate as G
    from mmada_parallel_b200.generators.stepwise import decode_text_with_masks
    from mmada_parallel_b200.schedule import stepwise_image_step_indices
    from mmada_parallel_b200.utils.image_utils import decode_vq_to_image, overlay_masked_cells
    import pytest
    g = torch.Generator().manual_seed(5)
    tok = G.PieceTokenizer()
    for n_mask_runs in range(6):
        ids = torch.randint(0, 126000, (1, 80), generator=g)
        for _ in range(n_mask_runs):
            a = int(torch.randint(0, 70, (1,), generator=g))
            ids[0, a:a + int(torch.randint(1, 25, (1,), generator=g))] = 126336
        assert decode_text_with_masks(ids, 5, 75, tok, 126336) == G.decode_text_with_masks(ids, 5, 75, tok, 126336)
    for T in (3, 10, 64, 100, 128):
        assert stepwise_image_step_indices(T) == G.stepwise_image_step_indices(T)

    class Dec:  # native decoder protocol: decode_code + decoder.upscale
        decoder = SimpleNamespace(upscale=16)

        def decode_code(self, ids, shape=None):
            h, w = shape
            x = torch.linspace(-1.2, 1.2, 3 * h * 16 * w * 16).view(1, 3, h * 16, w * 16)
            return x
    ids = torch.zeros(1, 4, dtype=torch.long)
    img = decode_vq_to_image(ids, None, None, 32, 32, Dec())
    want = ((Dec().decode_code(ids, (2, 2))[0] + 1) * 0.5).clamp(0, 1).permute(1, 2, 0).mul(255).round().to(torch.uint8)
    import numpy as np
    assert img.size == (32, 32) and np.array_equal(np.asarray(img), want.numpy())
    over = overlay_masked_cells(img, [1, 2], 2, 16, 16)
    diff = np.asarray(over).astype(int) - np.asarray(img).astype(int)
    assert (diff[:16, :16] == 0).all() and (diff[17:, 17:] == 0).all() and (diff[:15, 17:] != 0).any() and (diff[17:, :15] != 0).any()
    with pytest.raises(ValueError):
        decode_vq_to_image(torch.zeros(1, 5, dtype=torch.long), None, None, 32, 32, Dec())
    with pytest.raises(ValueError):
        decode_vq_to_image(ids, None, None, 32, 32, None)
    with pytest.raises(TypeError):
        decode_vq_to_image(ids, None, None, 32, 32, object())


def test_tensor_parallel_row_partition():
    """Rows of the residual stream owned per rank (tensor_parallel.row_partition): disjoint, in order, covering [0, M), owner
    of a row = row // rows_per_rank (what the GEMM's scatter epilogue evaluates), at most rows_per_rank rows each."""
    from mmada_parallel_b200.tensor_parallel import row_partition, rows_per_rank
    for M in (8, 9, 64, 77, 2414, 4682, 4096):
        for tp in (1, 2, 4, 8):
            R = rows_per_rank(M, tp)
            parts = [row_partition(M, tp, r) for r in range(tp)]
            assert parts[0][0] == 0 and sum(n for _, n in parts) == M
            for r, (r0, n) in enumerate(parts):
                assert 0 <= n <= R
                assert all(row // R == r for row in (r0, r0 + n - 1)) if n else True
    assert row_partition(2414, 8, 7) == (2114, 300)


def test_bench_workload_shapes_and_counts():
    """bench.py's synthetic input A is the SURVEY 8d layout (L = P + 2374 = 2414, image_start 1100, text span [2157, 2413)) and its
    FLOP count is the minimal-equivalent figure of BASELINE.md section 3 (7.101 PFLOP per sample); the CPU-arm protocol reports the
    host it ran on."""
    import bench
    lay = bench.synthetic_layout(seed=0)
    assert lay["input_ids"].shape == (1, 2414)
    assert (lay["image_start"], lay["text_start"], lay["text_end"]) == (1100, 2157, 2413)
    assert lay["uncon_text"].shape[1] == 1061 and lay["uncon_image"].shape[1] == 40
    assert int((lay["input_ids"] == bench.MASK).sum()) == 1024 + 256
    assert abs(bench.algorithmic_flops_per_sample(bench.MODEL_8B) / 1e15 - 7.101) < 0.002
    info = bench.host_cpu_info()
    assert 1 <= info["physical_cores"] <= info["logical_cpus"] and isinstance(info["model"], str)
    assert bench.load_peaks()[0] > 100


def test_tensor_parallel_chunk_split_and_half_m_unit_schedule():
    """chunk_split (row chunks of the pipelined tensor-parallel forward): one chunk below 1024 rows, else two chunks that cover
    [0, M), the first a multiple of 256 rows, chunk 1 never above half the rows (its buffers are sized for that) and every rank owns at
    least one row of each chunk up to TP=8."""
    from mmada_parallel_b200.tensor_parallel import chunk_split, row_partition
    assert chunk_split(1023) == [1023] and chunk_split(60) == [60]
    for M in (1024, 1500, 2341, 2414, 4682, 4828, 4096):
        parts = chunk_split(M)
        assert len(parts) == 2 and sum(parts) == M and parts[0] % 256 == 0 and 0 < parts[1] <= (M + 1) // 2
        for rows in parts:
            for tp in (2, 4, 8):
                assert row_partition(rows, tp, tp - 1)[1] >= 1
