"""Worker for tests/test_gpu_tp_batch.py::test_tensor_parallel_batch_two_gpus (launched with torchrun, one process per GPU): packed
forwards and generate_ti2ti_batch on the tensor-parallel model at TP = 2 (peer-memory collective) against the tp_size = 1 model,
and the ids of both ranks against each other."""
import contextlib
import io
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import load_golden, tiny_cfg_and_weights  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = f"cuda:{rank}"
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(dev))
from mmada_parallel_b200.generators.batch import generate_ti2ti_batch  # noqa: E402
from mmada_parallel_b200.tensor_parallel import TensorParallelLLaDA  # noqa: E402

t = load_golden("trajectory_a_tiny.pt")
cfg, sd = tiny_cfg_and_weights(t["meta"])
lay = t["layout"]
args = {k: lay[k] for k in ("text_start", "text_end", "image_start", "seq_len", "newline_every", "uncon_text", "uncon_image")}
ok = True
for precision in ("bf16", "fp8"):
    tp = TensorParallelLLaDA(cfg, sd, rank, world, max_seq_len=cfg.max_sequence_length, max_batch=3, device=dev, precision=precision)
    one = TensorParallelLLaDA(cfg, sd, 0, 1, max_seq_len=cfg.max_sequence_length, max_batch=3, device=dev, precision=precision)
    g = torch.Generator().manual_seed(11)
    lens = [150, 37, 201]
    ids = torch.randint(0, cfg.vocab_size, (sum(lens),), generator=g).to(dev)
    rows = torch.arange(0, sum(lens), dtype=torch.int32, device=dev)
    lg, _ = tp.forward_rows_packed(ids, lens, rows_a=rows)
    lg1, _ = one.forward_rows_packed(ids, lens, rows_a=rows)
    tol = 4 * lg1.float().abs().max().item() * 2.0 ** -8
    err = (lg.float() - lg1.float()).abs().max().item()
    res = [None] * world
    dist.all_gather_object(res, (err, tol))
    if rank == 0:
        print(f"{precision}: TP{world} packed logits vs tp_size=1 packed, max |dlogit| per rank {[round(x[0], 4) for x in res]} (tol {tol:.4f})")
    ok = ok and all(x[0] <= x[1] for x in res)
    reqs = []
    for i, (steps, ts) in enumerate([(8, 4), (6, 3)]):
        reqs.append(dict(input_ids=lay["input_ids"], text_steps=steps, timesteps=ts, text_gen_length=16, text_block_length=4,
                         temperature=1.0, text_temperature=0.0, cfg_scale=0.0, cfg_img=4.0,
                         generator=torch.Generator(device=dev).manual_seed(42 + i), **args))
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(5)
        out = generate_ti2ti_batch(tp, reqs)
    flat = torch.tensor([x for img, txt in out for x in img + txt], dtype=torch.int64, device=dev)
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    same_ids = all(torch.equal(gathered[0], x) for x in gathered)
    if rank == 0:
        print(f"{precision}: ranks produced identical generate_ti2ti_batch results: {same_ids}")
    ok = ok and same_ids
    dist.barrier()
    del tp, one
flag = torch.tensor([1 if ok else 0], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print("TP_BATCH_CHECK_OK" if int(flag.item()) == 1 else "TP_BATCH_CHECK_FAILED")
dist.destroy_process_group()
