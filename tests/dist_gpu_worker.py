"""Worker for tests/test_gpu_distributed.py: N ranks over NCCL, sharded multiply vs the oracle."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import matrel_b200 as mb  # noqa: E402
from matrel_b200.distributed import (GridGroups, GridPlan, ShardedMatrix, ingest_gate, pull_chunks, sharded_aggregate,  # noqa: E402
                                     sharded_elementwise, sharded_elementwise_any, sharded_multiply, sharded_multiply_allgather,
                                     sharded_multiply_overlapped, sharded_repartition, sharded_transpose, stream_barrier)
from oracle import matrel_oracle as O  # noqa: E402


def same_fp32(a, b):
    """Two fp32 products over DIFFERENT chunkings agree to fp32 rounding, not to the bit: each call centres and scales the operand
    blocks it sees, so the means (and with them the fp32 roundings of the centred values) depend on the call's extent.  Calls
    over the same extent are bit-identical (the sums behind the means and corrections are added in a fixed order)."""
    return float(np.max(np.abs(a - b))) <= 1e-5 * float(np.max(np.abs(b)))


def siblings(s, groups, A, planA, rank, device, n, k, blk):
    """The multiply's siblings on the same grid: transpose (one packed P2P exchange, flag flip), co-partitioned element-wise
    ops (no communication), aggregates (local kernel + one O(N) all-reduce)."""
    Af = O.rand_dense_dataset(n, k, blk, 42)
    full = O.assemble(Af, n, k, blk)
    AT = sharded_transpose(s, A)
    want = O.transpose(Af)
    got = {(b.rid, b.cid): b.matrix for b in AT.dataset.collect()}
    assert sorted(got) == sorted(AT.plan.owned(rank))
    for key, g in got.items():
        assert g.isTransposed and (g.numRows, g.numCols) == (want[key].numRows, want[key].numCols)
        assert np.array_equal(g.to_numpy(), want[key].to_numpy()), key
    A2 = ShardedMatrix.rand(s, planA, rank, 44, device)
    A2f = O.rand_dense_dataset(n, k, blk, 44)
    for op, fn in (("add", O.add_element), ("mul", O.multiply_element), ("div", O.divide_element)):
        w = fn(Af, n, k, A2f, n, k, blk)
        g = {(b.rid, b.cid): b.matrix for b in sharded_elementwise(op, A, A2, planA).collect()}
        assert sorted(g) == sorted(planA.owned(rank))
        for key, m in g.items():
            assert np.allclose(m.to_numpy(), w[key].to_numpy(), rtol=1e-14, atol=0), (op, key)
    # operands that start on DIFFERENT placement grids: A2 arrives in the RowPartitioner layout (world x 1); the element-wise
    # operator re-partitions it to A's grid (NCCL point-to-point all-to-all) and must give the co-partitioned result bit for bit
    world = planA.world
    A2_rows = sharded_repartition(s, A2, GridPlan(world, n, k, blk, world, 1))
    assert sorted(A2_rows.dataset.block_ids()) == sorted(A2_rows.plan.owned(rank))
    for op, fn in (("add", O.add_element), ("div", O.divide_element)):
        w = fn(Af, n, k, A2f, n, k, blk)
        res, keep_b = sharded_elementwise_any(op, s, A, A2_rows)
        g = {(b.rid, b.cid): b.matrix for b in res.collect()}
        assert sorted(g) == sorted(planA.owned(rank))
        for key, m in g.items():
            assert np.allclose(m.to_numpy(), w[key].to_numpy(), rtol=1e-14, atol=0), ("repartitioned", op, key)
    r, c = planA.coords(rank)
    rows = np.concatenate([np.arange(i * blk, min(n, (i + 1) * blk)) for i in range(r, planA.nbr, planA.pr)])
    cols = np.concatenate([np.arange(j * blk, min(k, (j + 1) * blk)) for j in range(c, planA.nbc, planA.pc)])
    assert np.allclose(sharded_aggregate("rowSum", groups, A), full.sum(axis=1)[rows], rtol=1e-12)
    assert np.allclose(sharded_aggregate("colSum", groups, A), full.sum(axis=0)[cols], rtol=1e-12)
    assert abs(sharded_aggregate("sum", groups, A) - full.sum()) <= 1e-12 * full.sum()
    if n == k:
        assert abs(sharded_aggregate("trace", groups, A) - np.trace(full)) <= 1e-12 * abs(np.trace(full))


def main():
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", device_id=device)
    rank, world = dist.get_rank(), dist.get_world_size()
    for (n, k, m, blk) in [(1024, 1024, 1024, 128), (7 * 64 - 6, 5 * 64, 6 * 64 - 10, 64)]:
        planA, planB, planC = GridPlan(world, n, k, blk), GridPlan(world, k, m, blk), GridPlan(world, n, m, blk)
        groups = GridGroups(planA, rank)
        stream = torch.cuda.Stream(device=device)
        with torch.cuda.stream(stream):
            algo = int(os.environ.get("MATREL_GEMM_ALGO", "0"))
            s = mb.MatfastSession(device=local_rank, stream=stream.cuda_stream, gemm_algo=algo)
            A = ShardedMatrix.rand(s, planA, rank, 42, device)
            B = ShardedMatrix.rand(s, planB, rank, 43, device)
            # the product path: peer pulls over CUDA IPC (copy engines), chunked and overlapped with the multiply
            s.sync()
            dist.barrier()
            dC, keep = sharded_multiply(s, groups, A, B, planA, planB, nchunks=3)
            got = {(b.rid, b.cid): b.matrix for b in dC.collect()}
            s_launches = s.stats()["kernel_launches"]
            assert world == 1 or s.stats()["p2p_bytes"] > 0
            # the NCCL all-gather form must give the same blocks (bit for bit: same kernels, same summation order)
            dG, keepG = sharded_multiply_allgather(s, groups, A, B, planA, planB)
            gotG = {(b.rid, b.cid): b.matrix for b in dG.collect()}
            assert sorted(gotG) == sorted(got)
            for key in got:   # (the fp32 path centres per call: equal to rounding where the chunkings differ, see same_fp32)
                assert np.array_equal(gotG[key].values, got[key].values) if algo != 3 else same_fp32(gotG[key].values, got[key].values), key
            # operands that arrive from the HOST into sharded datasets (put_block on the ingest stream), barrier, pull, multiply
            from matrel_b200.dataset import create_sharded
            Ah = O.rand_dense_dataset(n, k, blk, 42)
            Bh = O.rand_dense_dataset(k, m, blk, 43)
            eA = ShardedMatrix(planA, rank, torch.zeros_like(A.slab), None, s)
            eB = ShardedMatrix(planB, rank, torch.zeros_like(B.slab), None, s)
            eA.peer_slabs(); eB.peer_slabs()
            mk = lambda H, i, j: mb.MatrixBlock(i, j, mb.DenseMatrix(H[(i, j)].numRows, H[(i, j)].numCols, H[(i, j)].values))  # noqa: E731
            side, tick = torch.cuda.Stream(device=device), torch.zeros(1, device=device)
            first = None
            for rep in range(3):
                if rep < 2:     # upload everything, wait, barrier, multiply
                    eA.sharded.put_blocks(mk(Ah, i, j) for (i, j) in planA.owned(rank))
                    eB.sharded.put_blocks(mk(Bh, i, j) for (i, j) in planB.owned(rank))
                    s.wait_ingest()
                    stream_barrier(device)
                    dE, keepE = sharded_multiply(s, groups, eA, eB, planA, planB, nchunks=2)
                else:           # pipelined: pieces of A's block rows and B's block columns uploaded alternately, one gate event each
                    nch, crow, ccol = pull_chunks(planA, planB, rank, 3)
                    evs = []
                    for ch in range(nch):
                        eA.sharded.put_blocks(mk(Ah, i, j) for (i, j) in planA.owned(rank) if i in crow[ch])
                        evs.append(ingest_gate(s, side, tick))
                        eB.sharded.put_blocks(mk(Bh, i, j) for (i, j) in planB.owned(rank) if j in ccol[ch])
                        evs.append(ingest_gate(s, side, tick))
                    dE, keepE = sharded_multiply(s, groups, eA, eB, planA, planB, nchunks=nch, gates=[e.cuda_event for e in evs])
                gotE = {(b.rid, b.cid): b.matrix for b in dE.collect()}
                stream_barrier(device)
                assert sorted(gotE) == sorted(got)
                for key in got:
                    assert np.array_equal(gotE[key].values, got[key].values) if algo != 3 else same_fp32(gotE[key].values, got[key].values), (rep, key)
                if rep == 0:
                    first = {key: x.values.copy() for key, x in gotE.items()}
                elif rep == 1:    # the same chunking as rep 0: the same extents, so bit for bit on every path
                    for key in got:
                        assert np.array_equal(gotE[key].values, first[key]), (rep, key)
            # the overlapped exchange (A gathered in chunks on a side stream) must give the same blocks
            outs, keep2 = sharded_multiply_overlapped(s, groups, A, B, planA, planB, torch.cuda.Stream(device=device), nchunks=3)
            got2 = {(b.rid, b.cid): b.matrix for d in outs for b in d.collect()}
            assert sorted(got2) == sorted(got)
            for key in got:
                assert np.array_equal(got2[key].values, got[key].values) if algo != 3 else same_fp32(got2[key].values, got[key].values), key
            if algo in (0, 1):
                siblings(s, groups, A, planA, rank, device, n, k, blk)
            s.stop()
        want = O.matrix_multiply(O.rand_dense_dataset(n, k, blk, 42), n, k, O.rand_dense_dataset(k, m, blk, 43), k, m, blk)
        assert sorted(got) == sorted(planC.owned(rank)), (rank, sorted(got))
        for key, g in got.items():
            w = want[key]
            assert (g.numRows, g.numCols, g.isTransposed) == (w.numRows, w.numCols, False)
            err = float(np.max(np.abs(g.values - w.values)) / np.max(np.abs(w.values)))
            assert err <= (1e-5 if algo == 3 else 1e-12), (key, err)      # algo 3 = fp32 results (3xTF32)
        if algo == 2:
            assert s_launches >= 8, s_launches     # absmax/slice passes + one GEMM per diagonal: the tensor-core path really ran
        if algo == 4:
            assert s_launches >= 7, s_launches     # absmax x2, exp, residues x2, one GEMM launch over all moduli, CRT
        cnt = torch.tensor([len(got)], dtype=torch.int64, device=device)
        dist.all_reduce(cnt)
        assert int(cnt.item()) == len(want)
    dist.barrier()
    if rank == 0:
        print(f"OK world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
