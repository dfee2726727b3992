"""Worker for tests/test_gpu_tp_fp8.py::test_tensor_parallel_fp8_two_gpus (launched with torchrun, one process per GPU): the
FP8 tensor-parallel model at TP = 2 (multi-head and h4_kv2_bias) against the tp_size = 1 FP8 model, the NCCL collective, itself,
and across ranks, and the ids of a short generation."""
import contextlib
import io
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import load_golden  # noqa: E402
from oracle import llada_gqa  # noqa: E402  (tests may use the oracle's seeded weight generator)

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = f"cuda:{rank}"
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
from mmada_parallel_b200.generators.parallel_generator import generate_ti2ti  # noqa: E402
from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA  # noqa: E402

g = load_golden("forward_gqa_tiny.pt")
lay = g["layout"]
ids = g["ids"].to(dev)
args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
ok = True


def run_ids(model):
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(5)
        img, txt = generate_ti2ti(model, g["ids"], text_steps=8, timesteps=4, text_gen_length=16, text_block_length=4, temperature=1.0,
                                  text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0, generator=torch.Generator(device=dev).manual_seed(42), **args)
    return img + txt


for name in ("h4_kv2_bias", "h4_mqa"):
    cfg = llada_gqa.make_config(**g["meta"]["common"], **g["configs"][name]["config"])
    sd = llada_gqa.make_weights(cfg, seed=g["meta"]["weight_seed"])
    kw = dict(max_seq_len=cfg.max_sequence_length, max_batch=3, device=dev, precision="fp8")
    tp = TensorParallelLLaDA(cfg, sd, rank, world, **kw)
    tp_nccl = TensorParallelLLaDA(cfg, sd, rank, world, collective="nccl", **kw)
    lg = tp(ids).logits
    lg_nccl = tp_nccl(ids).logits
    rep = torch.equal(tp(ids).logits, lg)
    one = TensorParallelLLaDA(cfg, sd, 0, 1, **kw)       # tp_size = 1 on this GPU: no collective
    lg_1 = one(ids).logits
    tol = 4 * lg_1.float().abs().max().item() * 2.0 ** -8
    err1 = (lg.float() - lg_1.float()).abs().max().item()
    err_n = (lg.float() - lg_nccl.float()).abs().max().item()
    res = [None] * world
    dist.all_gather_object(res, (err1, err_n, tol, rep))
    if rank == 0:
        print(f"{name}: TP{world} fp8 vs tp_size=1 fp8 max |dlogit| {[round(x[0], 4) for x in res]}, vs nccl {[round(x[1], 4) for x in res]} "
              f"(tol {tol:.4f}), repeatable {[x[3] for x in res]}")
    ok = ok and all(x[3] and x[0] <= x[2] and x[1] <= x[2] for x in res)
    ref = lg.clone()
    dist.broadcast(ref, src=0)
    same = torch.tensor([1 if torch.equal(ref, lg) else 0], device=dev)
    dist.all_reduce(same, op=dist.ReduceOp.MIN)
    ok = ok and int(same.item()) == 1
    t = torch.tensor(run_ids(tp), dtype=torch.int64, device=dev)
    t1 = torch.tensor(run_ids(one), dtype=torch.int64, device=dev)
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    same_ids = all(torch.equal(gathered[0], x) for x in gathered)
    agree = float((t == t1).float().mean().item())
    if rank == 0:
        print(f"{name}: ranks produced identical token sequences: {same_ids}; ids equal to tp_size=1 fp8: {agree:.3f}")
    ok = ok and same_ids and agree >= 0.9
    dist.barrier()
    del tp, tp_nccl, one
flag = torch.tensor([1 if ok else 0], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print("TP_FP8_CHECK_OK" if int(flag.item()) == 1 else "TP_FP8_CHECK_FAILED")
dist.destroy_process_group()
