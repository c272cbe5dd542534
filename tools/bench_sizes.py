"""Sharded dense multiply at any north-star size / precision on the GPUs of one box (1 process per GPU; also runs with 1 GPU).
   [torchrun --nproc-per-node P] tools/bench_sizes.py N BLK ALGO [steps] [PRxPC]
ALGO: 0 = auto (wgmma Ozaki-II, fp64-equivalent), 1 = fp64 DMMA, 3 = fp32 (wgmma tf32, 3xTF32; BASELINE configs[3]).
Prints one JSON line on rank 0: ms (max over ranks, device-timed), TFLOP/s, fraction of the measured roof, and the error of one
sampled output block per rank against numpy fp64 on the host (fp32-rounded inputs for ALGO 3), MAX over ranks."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import matrel_b200 as mb
from matrel_b200.dataset import memcpy_d2h
from matrel_b200.distributed import GridGroups, GridPlan, ShardedMatrix, sharded_multiply

n, blk, algo = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
steps = int(sys.argv[4]) if len(sys.argv) > 4 else 3
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
local_rank = int(os.environ.get("LOCAL_RANK", "0"))
device = torch.device("cuda", local_rank)
torch.cuda.set_device(device)
dist = None
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=device)
if len(sys.argv) > 5:
    pr, pc = (int(x) for x in sys.argv[5].split("x"))
    plan = GridPlan(world, n, n, blk, pr, pc)
else:
    plan = GridPlan(world, n, n, blk)
nb = n // blk


def allmax(x):
    if world == 1:
        return float(x)
    t = torch.tensor([float(x)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def barrier():
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()


class _G:
    pass


groups = _G()
groups.rank = rank
stream = torch.cuda.Stream(device=device)
with torch.cuda.stream(stream):
    s = mb.MatfastSession(device=local_rank, stream=stream.cuda_stream, gemm_algo=algo)
    A = ShardedMatrix.rand(s, plan, rank, 42, device)
    B = ShardedMatrix.rand(s, plan, rank, 43, device)
    s.sync()
    pa, pb = A.peer_slabs(), B.peer_slabs()
    barrier()
    for _ in range(2):
        out = sharded_multiply(s, groups, A, B, plan, plan)
        del out
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        out = sharded_multiply(s, groups, A, B, plan, plan)
        del out
    e1.record(stream)
    barrier()
    ms = allmax(e0.elapsed_time(e1) / steps)
    dC, keep = sharded_multiply(s, groups, A, B, plan, plan)
    mine = plan.owned(rank)
    i, j = mine[(len(mine) * 2) // 3]
    rnd = (lambda x: x.astype(np.float32).astype(np.float64)) if algo == 3 else (lambda x: x)
    sub = min(blk, 256)                                     # a 256 x 256 corner of the block keeps the host product cheap
    want = np.zeros((sub, sub))
    bufa, bufb = np.empty(blk * blk), np.empty(blk * blk)
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=8, user_api="blas"):
        for k in range(nb):
            memcpy_d2h(s, pa[plan.owner(i, k)] + plan.slot(i, k) * plan.slot_elems * 8, bufa)
            memcpy_d2h(s, pb[plan.owner(k, j)] + plan.slot(k, j) * plan.slot_elems * 8, bufb)
            want += rnd(bufa.reshape(blk, blk).T[:sub]) @ rnd(bufb.reshape(blk, blk).T[:, :sub])
    got = dC.get_block(i, j).to_numpy()[:sub, :sub]
    err = allmax(float(np.max(np.abs(got - want)) / np.max(np.abs(want))))
    st = s.stats()
    del dC, keep
    barrier()
    s.stop()
if rank == 0:
    tflops = 2.0 * n ** 3 / (ms * 1e-3) / 1e12
    line = {"config": f"{n}x{n} {'fp32' if algo == 3 else 'fp64'} dense multiply, {blk}-block, {plan.pr}x{plan.pc} grid over {world}xH100",
            "algo": {0: "auto: wgmma Ozaki-II (int8 residues + CRT), fp64-equivalent", 1: "fp64 DMMA (mma.sync m8n8k4)",
                     3: "wgmma tf32, 3xTF32 split, mean-centred, fp64 re-accumulation of 2048-deep K chunks"}.get(algo, str(algo)),
            "n_gpus": world, "ms_per_step": ms, "TFLOPs": tflops, "max_rel_err_sampled_blocks": err, "tc_path": bool(st["tc_gemm_launches"])}
    if algo == 3:
        line["raw_tf32_TFLOPs"] = 3 * tflops
        line["frac_of_datasheet_tf32"] = 3 * tflops / (world * 495.0)    # H100 SXM data sheet, dense TF32 (not measured)
    if algo in (0, 1):
        line["x_datasheet_fp64_tensor"] = tflops / (world * 67.0)        # H100 SXM data sheet, FP64 tensor core (not measured)
    print(json.dumps(line), flush=True)
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
