"""Worker for tests/test_gpu_tp_gqa.py::test_tensor_parallel_gqa_two_gpus (launched with torchrun, one process per GPU): the
tensor-parallel model on the reference fixture's grouped-query configs h4_kv2_bias (each rank owns one of the 2 kv heads) and
h4_mqa (the one kv head computed on both ranks) against the single-GPU model, the NCCL collective, itself, and across ranks."""
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
from mmada_parallel_b200.model import LLaDAForMultiModalGeneration  # noqa: E402
from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA  # noqa: E402

g = load_golden("forward_gqa_tiny.pt")
lay = g["layout"]
ids = g["ids"].to(dev)
args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
ok = True
for name in ("h4_kv2_bias", "h4_mqa"):
    cfg = llada_gqa.make_config(**g["meta"]["common"], **g["configs"][name]["config"])
    sd = llada_gqa.make_weights(cfg, seed=g["meta"]["weight_seed"])
    tp = TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=cfg.max_sequence_length, max_batch=3, device=dev)
    tp_nccl = TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=cfg.max_sequence_length, max_batch=3, device=dev, collective="nccl")
    lg = tp(ids).logits
    lg_nccl = tp_nccl(ids).logits
    tol = 4 * lg.float().abs().max().item() * 2.0 ** -8
    d_modes = (lg.float() - lg_nccl.float()).abs().max().item()
    rep = torch.equal(tp(ids).logits, lg)
    res = [None] * world
    dist.all_gather_object(res, (d_modes, tol, rep))
    if rank == 0:
        print(f"{name}: p2p vs nccl max |dlogit| per rank {[round(x[0], 4) for x in res]} (tol {tol:.4f}), repeatable {[x[2] for x in res]}")
        ok = ok and all(x[2] and x[0] <= x[1] for x in res)
    ref = lg.clone()
    dist.broadcast(ref, src=0)
    same = torch.tensor([1 if torch.equal(ref, lg) else 0], device=dev)
    dist.all_reduce(same, op=dist.ReduceOp.MIN)
    ok = ok and int(same.item()) == 1
    if rank == 0:
        single = LLaDAForMultiModalGeneration(cfg, max_seq_len=cfg.max_sequence_length, max_batch=1, device=dev)
        single.load_state_dict(sd)
        lg_1 = single(ids, infer=True).logits
        err = (lg.float() - lg_1.float()).abs().max().item()
        tol1 = 4 * lg_1.float().abs().max().item() * 2.0 ** -8
        print(f"{name}: TP{world} vs single GPU max err {err:.4f} (tol {tol1:.4f}), identical on all ranks {bool(same.item())}")
        ok = ok and err <= tol1
        del single
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(5)
        img, txt = generate_ti2ti(tp, g["ids"], text_steps=8, timesteps=4, text_gen_length=16, text_block_length=4, temperature=1.0,
                                  text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0, generator=torch.Generator(device=dev).manual_seed(42), **args)
    t = torch.tensor(img + txt, dtype=torch.int64, device=dev)
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    same_ids = all(torch.equal(gathered[0], x) for x in gathered)
    if rank == 0:
        print(f"{name}: ranks produced identical token sequences: {same_ids}")
    ok = ok and same_ids
    dist.barrier()
    del tp, tp_nccl
flag = torch.tensor([1 if ok else 0], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print("TP_GQA_CHECK_OK" if int(flag.item()) == 1 else "TP_GQA_CHECK_FAILED")
dist.destroy_process_group()
