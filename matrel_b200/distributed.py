"""Grid-partitioned block multiply across the GPUs of one box: one process per GPU,
``torch.distributed`` for the plumbing (rendezvous, barriers, IPC handle exchange, small reductions), the
engine's own C ABI for the data path: every rank PULLS the operand blocks it needs straight out of its
peers' device slabs over NVLink / NVSwitch with the copy engines (CUDA IPC mappings, ``mr_grid_multiply``),
block row by block row, while its own sm_90a kernels already multiply what has arrived.

What it replaces in the reference (M/ = <reference>/src/main/scala/org/apache/spark/sql/matfast/):
  * the 2 x groupByKey + join that co-locate A(:, k) with B(k, :) (M/execution/MatfastExecutionHelper.scala:236-249)
    -> chunked peer pulls of A along the grid row and of B along the grid column, overlapped with the multiply
    (``sharded_multiply``; the NCCL all-gather form is kept as ``sharded_multiply_allgather``);
  * reduceByKey(LocalMatrix.add) (:255) -> nothing: the layout is C-stationary, every rank owns whole
    output blocks and keeps the full K reduction inside the GEMM kernel's accumulators;
  * RowPartitioner / ColumnPartitioner placement (M/partitioner/RowPartitioner.scala:34,
    ColumnPartitioner.scala:34): rank (r, c) of the pr x pc grid owns blocks with rid % pr == r and
    cid % pc == c, for A, B and C alike.

Nothing in the planning half of this module needs a GPU (``GridPlan``, ``gather_panels`` work on CPU
tensors over gloo), which is how tests/test_distributed_cpu.py covers the N > 1 path.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

GRID_SHAPES = {1: (1, 1), 2: (1, 2), 4: (2, 2), 8: (2, 4)}


def grid_shape(world: int) -> Tuple[int, int]:
    if world in GRID_SHAPES:
        return GRID_SHAPES[world]
    pr = int(world ** 0.5)
    while world % pr:
        pr -= 1
    return pr, world // pr


@dataclass
class GridPlan:
    """Placement arithmetic of an nrows x ncols block matrix on a pr x pc process grid."""
    world: int
    nrows: int
    ncols: int
    blk: int
    pr: int = 0
    pc: int = 0

    def __post_init__(self):
        if not self.pr:
            self.pr, self.pc = grid_shape(self.world)
        assert self.pr * self.pc == self.world
        self.nbr = -(-self.nrows // self.blk)
        self.nbc = -(-self.ncols // self.blk)
        self.slots_r = -(-self.nbr // self.pr)
        self.slots_c = -(-self.nbc // self.pc)
        self.slot_elems = self.blk * self.blk

    def coords(self, rank: int) -> Tuple[int, int]:
        return rank // self.pc, rank % self.pc

    def rank_of(self, r: int, c: int) -> int:
        return r * self.pc + c

    def owner(self, rid: int, cid: int) -> int:
        """RowPartitioner x ColumnPartitioner: (rid % pr, cid % pc)."""
        return self.rank_of(rid % self.pr, cid % self.pc)

    def slot(self, rid: int, cid: int) -> int:
        """Index of block (rid, cid) inside its owner's slab."""
        return (rid // self.pr) * self.slots_c + (cid // self.pc)

    @property
    def local_slots(self) -> int:
        return self.slots_r * self.slots_c

    def block_shape(self, rid: int, cid: int) -> Tuple[int, int]:
        return (min(self.blk, self.nrows - rid * self.blk), min(self.blk, self.ncols - cid * self.blk))

    def owned(self, rank: int) -> List[Tuple[int, int]]:
        r, c = self.coords(rank)
        return [(i, j) for i in range(r, self.nbr, self.pr) for j in range(c, self.nbc, self.pc)]

    def row_group_ranks(self, rank: int) -> List[int]:
        r, _ = self.coords(rank)
        return [self.rank_of(r, c) for c in range(self.pc)]

    def col_group_ranks(self, rank: int) -> List[int]:
        _, c = self.coords(rank)
        return [self.rank_of(r, c) for r in range(self.pr)]


class GridGroups:
    """Row / column sub-communicators (every rank must construct this collectively)."""

    def __init__(self, plan: GridPlan, rank: int):
        import torch.distributed as dist
        self.plan, self.rank = plan, rank
        self.row_group = self.col_group = None
        for r in range(plan.pr):
            ranks = [plan.rank_of(r, c) for c in range(plan.pc)]
            g = dist.new_group(ranks) if len(ranks) > 1 else None
            if rank in ranks:
                self.row_group = g
        for c in range(plan.pc):
            ranks = [plan.rank_of(r, c) for r in range(plan.pr)]
            g = dist.new_group(ranks) if len(ranks) > 1 else None
            if rank in ranks:
                self.col_group = g


def gather_panels(local_slab, group, nranks: int):
    """All-gather equal-sized slabs [local_slots, slot_elems] -> [nranks, local_slots, slot_elems].
    (The reference moves the same blocks through groupByKey + join.)"""
    import torch
    import torch.distributed as dist
    if nranks == 1 or group is None:
        return local_slab.unsqueeze(0)
    flat = torch.empty((nranks * local_slab.shape[0],) + tuple(local_slab.shape[1:]), dtype=local_slab.dtype,
                       device=local_slab.device)
    dist.all_gather_into_tensor(flat, local_slab.contiguous(), group=group)
    return flat.view((nranks,) + tuple(local_slab.shape))


def panel_blocks_A(plan: GridPlan, rank: int):
    """(rid, k, source index in the row group, slot) for every A block this rank needs: all k of its rows."""
    r, _ = plan.coords(rank)
    kplan = GridPlan(plan.world, plan.nrows, plan.ncols, plan.blk, plan.pr, plan.pc)
    return [(i, k, k % plan.pc, kplan.slot(i, k)) for i in range(r, plan.nbr, plan.pr) for k in range(plan.nbc)]


def panel_blocks_B(plan: GridPlan, rank: int):
    """(k, cid, source index in the column group, slot) for every B block this rank needs: all k of its columns."""
    _, c = plan.coords(rank)
    return [(k, j, k % plan.pr, plan.slot(k, j)) for k in range(plan.nbr) for j in range(c, plan.nbc, plan.pc)]


class ShardedMatrix:
    """The blocks of one matrix that this rank owns, in one contiguous device slab (torch tensor).

    ``dataset`` registers the owned blocks as an ordinary Dataset (borrowed windows of the slab); ``sharded`` is the same slab
    adopted as a sharded dataset of the C ABI (``mr_matrix_adopt_sharded``), the operand type of ``mr_grid_multiply``."""

    def __init__(self, plan: GridPlan, rank: int, slab, dataset=None, session=None, transposed: bool = False):
        self.plan, self.rank, self.slab, self.dataset = plan, rank, slab, dataset
        self.session = session if session is not None else (dataset.matfastSession if dataset is not None else None)
        self.transposed = transposed
        self._sharded = None
        self._peers = None

    @staticmethod
    def rand(session, plan: GridPlan, rank: int, seed0: int, device) -> "ShardedMatrix":
        import torch
        from .dataset import rand_partition
        slab = torch.zeros((plan.local_slots, plan.slot_elems), dtype=torch.float64, device=device)
        r, c = plan.coords(rank)
        ds = rand_partition(session, plan.nrows, plan.ncols, plan.blk, seed0, plan.pr, plan.pc, r, c,
                            slab.data_ptr(), plan.slot_elems)
        return ShardedMatrix(plan, rank, slab, ds, session)

    @property
    def sharded(self):
        if self._sharded is None:
            from .dataset import adopt_sharded
            r, c = self.plan.coords(self.rank)
            self._sharded = adopt_sharded(self.session, self.plan.nrows, self.plan.ncols, self.plan.blk, self.plan.pr, self.plan.pc,
                                          r, c, self.slab.data_ptr(), self.transposed)
        return self._sharded

    def peer_slabs(self) -> List[int]:
        """Device pointers, valid in THIS process, of every rank's slab of this matrix (collective: every rank must call it).
        The peers' allocations are mapped through CUDA IPC once and cached."""
        if self._peers is None:
            import torch.distributed as dist
            from .dataset import ipc_export, ipc_open
            mine = ipc_export(self.slab.data_ptr())
            if dist.is_initialized() and dist.get_world_size() > 1:
                everyone = [None] * dist.get_world_size()
                dist.all_gather_object(everyone, mine)
            else:
                everyone = [mine]
            self._peers = [self.slab.data_ptr() if q == self.rank else ipc_open(self.session, h, off)
                           for q, (h, off) in enumerate(everyone)]
        return self._peers


def sharded_multiply(session, groups: GridGroups, A: ShardedMatrix, B: ShardedMatrix, planA: GridPlan, planB: GridPlan,
                     nchunks: int = 4, gates=None):
    """C = A * B, C-stationary on the process grid, through ``mr_grid_multiply``: this rank pulls A(i, :) of its block rows from
    the ranks of its grid row and B(:, j) of its block columns from its grid column out of their slabs (copy engines over
    NVLink, ``nchunks`` pieces of A's block rows and of B's block columns, fetched alternately) while the multiply already runs
    on the corner of C that the pieces landed so far unlock.
    The peers' slabs must be complete when the pulls run and stay untouched until every rank's multiply has consumed them:
    callers that rewrite slabs between steps put a stream barrier around the call (``stream_barrier``).
    Returns (local C Dataset -- a sharded dataset --, keep-alive objects)."""
    from .dataset import grid_multiply
    rank = groups.rank
    r, c = planA.coords(rank)
    pa, pb = A.peer_slabs(), B.peer_slabs()
    rowA = [pa[planA.rank_of(r, cc)] for cc in range(planA.pc)]
    colB = [pb[planB.rank_of(rr, c)] for rr in range(planB.pr)]
    dC = grid_multiply(session, A.sharded, B.sharded, rowA, colB, nchunks, gates)
    return dC, (A, B)


def pull_chunks(planA: GridPlan, planB: GridPlan, rank: int, nchunks: int):
    """The pieces ``mr_grid_multiply`` cuts this rank's pull into: (nchunks, [global block-row ids of A per piece], [global
    block-column ids of B per piece]); piece ch of A is fetched before piece ch of B, pieces may be empty."""
    r, c = planA.coords(rank)
    rows = list(range(r, planA.nbr, planA.pr))
    cols = list(range(c, planB.nbc, planB.pc))
    nchunks = max(1, min(nchunks, 64))
    cut = lambda v: [v[len(v) * ch // nchunks:len(v) * (ch + 1) // nchunks] for ch in range(nchunks)]  # noqa: E731
    return nchunks, cut(rows), cut(cols)


def ingest_gate(session, side, tick):
    """'Every rank's host->device copies submitted so far have landed', as a CUDA event: the side stream waits for this rank's
    ingest, runs a one-element all-reduce (complete only when every rank has got there), and the event recorded behind it is
    what ``mr_grid_multiply_gated`` lets the pull of a piece wait for.  No host synchronisation."""
    import torch
    import torch.distributed as dist
    session.wait_ingest_on(side.cuda_stream)
    with torch.cuda.stream(side):
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(tick)
        ev = torch.cuda.Event()
        ev.record(side)
    return ev


def stream_barrier(device):
    """All ranks have reached this point of their CURRENT CUDA streams (a one-element NCCL all-reduce; no host sync)."""
    import torch
    import torch.distributed as dist
    if dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.zeros(1, device=device)
        dist.all_reduce(t)


def sharded_multiply_allgather(session, groups: GridGroups, A: ShardedMatrix, B: ShardedMatrix, planA: GridPlan, planB: GridPlan):
    """C = A * B, C-stationary on the process grid, with NCCL all-gathers of the operand slabs (the first form benchmarked;
    kept for comparison and for ranks that cannot map their peers' memory).  Returns (local C Dataset, keep-alive tensors).

    planA describes A (n x k), planB describes B (k x m); both share blk and the grid."""
    from .dataset import Dataset
    rank = groups.rank
    pr, pc = planA.pr, planA.pc
    gA = gather_panels(A.slab, groups.row_group, pc)      # [pc, slots, elems]: A(i, :) for my rows
    gB = gather_panels(B.slab, groups.col_group, pr)      # [pr, slots, elems]: B(:, j) for my columns
    esz = 8
    baseA, strideA0, strideA1 = gA.data_ptr(), gA.stride(0) * esz, gA.stride(1) * esz
    baseB, strideB0, strideB1 = gB.data_ptr(), gB.stride(0) * esz, gB.stride(1) * esz
    dA = session.emptyDataset()
    blocks = panel_blocks_A(planA, rank)
    shapes = [planA.block_shape(i, k) for i, k, _, _ in blocks]
    dA.put_blocks_device([b[0] for b in blocks], [b[1] for b in blocks], [s[0] for s in shapes], [s[1] for s in shapes],
                         [baseA + src * strideA0 + slot * strideA1 for _, _, src, slot in blocks])
    dB = session.emptyDataset()
    blocks = panel_blocks_B(planB, rank)
    shapes = [planB.block_shape(k, j) for k, j, _, _ in blocks]
    dB.put_blocks_device([b[0] for b in blocks], [b[1] for b in blocks], [s[0] for s in shapes], [s[1] for s in shapes],
                         [baseB + src * strideB0 + slot * strideB1 for _, _, src, slot in blocks])
    dC = dA.matrixMultiply(planA.nrows, planA.ncols, dB, planB.nrows, planB.ncols, planA.blk)
    return dC, (gA, gB, dA, dB)


def sharded_multiply_overlapped(session, groups: GridGroups, A: ShardedMatrix, B: ShardedMatrix, planA: GridPlan,
                                planB: GridPlan, comm_stream, nchunks: int = 4):
    """Same result as :func:`sharded_multiply`, with the A exchange pipelined against the GEMM: B and the first
    chunk of A's block rows are gathered up front; while the kernel multiplies chunk c on the compute stream, NCCL
    gathers chunk c+1 on `comm_stream`.  Returns (list of local C Datasets -- one per chunk --, keep-alive objects)."""
    import torch
    rank = groups.rank
    pr, pc = planA.pr, planA.pc
    compute = torch.cuda.current_stream()
    r, _ = planA.coords(rank)
    my_rows = list(range(r, planA.nbr, pr))
    nchunks = max(1, min(nchunks, len(my_rows)))
    bounds = [len(my_rows) * c // nchunks for c in range(nchunks + 1)]
    esz = 8
    comm_stream.wait_stream(compute)                       # the slabs were produced on the compute stream
    events, gathered = [], []
    with torch.cuda.stream(comm_stream):
        gB = gather_panels(B.slab, groups.col_group, pr)
        for c in range(nchunks):
            lo, hi = bounds[c], bounds[c + 1]
            # block rows are contiguous in the slab: slots [(i // pr) * slots_c, ...)
            part = A.slab[lo * planA.slots_c:hi * planA.slots_c]
            gathered.append(gather_panels(part, groups.row_group, pc))
            ev = torch.cuda.Event()
            ev.record(comm_stream)
            events.append(ev)
    dB = session.emptyDataset()
    blocks = panel_blocks_B(planB, rank)
    shapes = [planB.block_shape(k, j) for k, j, _, _ in blocks]
    baseB, sB0, sB1 = gB.data_ptr(), gB.stride(0) * esz, gB.stride(1) * esz
    dB.put_blocks_device([b[0] for b in blocks], [b[1] for b in blocks], [x[0] for x in shapes], [x[1] for x in shapes],
                         [baseB + src * sB0 + slot * sB1 for _, _, src, slot in blocks])
    outs, keep = [], [gB, dB]
    for c in range(nchunks):
        lo, hi = bounds[c], bounds[c + 1]
        gA = gathered[c]
        base, s0, s1 = gA.data_ptr(), gA.stride(0) * esz, gA.stride(1) * esz
        dA = session.emptyDataset()
        rids, cids, nr, nc, ptrs = [], [], [], [], []
        for li in range(lo, hi):
            i = my_rows[li]
            for k in range(planA.nbc):
                rr, cc = planA.block_shape(i, k)
                rids.append(i); cids.append(k); nr.append(rr); nc.append(cc)
                ptrs.append(base + (k % pc) * s0 + ((li - lo) * planA.slots_c + k // pc) * s1)
        dA.put_blocks_device(rids, cids, nr, nc, ptrs)
        compute.wait_event(events[c])
        outs.append(dA.matrixMultiply(planA.nrows, planA.ncols, dB, planB.nrows, planB.ncols, planA.blk))
        keep += [gA, dA]
    for g in gathered:                                     # the caching allocator must not recycle them under the GEMM
        g.record_stream(compute)
    gB.record_stream(compute)
    return outs, keep


# --------------------------------------------------------------------------------------------------
# bench.py's N > 1 arm
# --------------------------------------------------------------------------------------------------
# ---- the siblings of the multiply on the same grid -------------------------------------------------------------------
def sharded_elementwise(op: str, A: ShardedMatrix, B: ShardedMatrix, plan: GridPlan):
    """add / mul / div of two matrices laid out on the SAME grid.  Both sides are co-partitioned (RowPartitioner x
    ColumnPartitioner arithmetic on A and B alike), which is the reference's `zipPartitions` fast path
    (M/execution/MatfastExecutionHelper.scala:64-105 / :107-139 / :141-173 when the partitioners match): no communication, each
    rank runs the element-wise kernel on its own blocks.  Returns the local result Dataset."""
    fn = {"add": "addElement", "mul": "multiplyElement", "div": "divideElement"}[op]
    return getattr(A.dataset, fn)(plan.nrows, plan.ncols, B.dataset, plan.nrows, plan.ncols, plan.blk)


def repartition_routes(src: GridPlan, dst: GridPlan, rank: int):
    """Block moves of repartitionWithTargetPartitioner (M/execution/MatfastExecutionHelper.scala:34-44) between two placement grids
    of the same ranks (e.g. (P, 1) = RowPartitioner, (1, P) = ColumnPartitioner, (pr, pc) = the multiply's grid): block (i, j) moves
    from src.owner(i, j) to dst.owner(i, j).  Returns (sends, recvs): sends[peer] = [(src_slot, dst_slot)], recvs[peer] = [dst_slot],
    both ordered by block id so that one packed message per peer suffices."""
    assert (src.world, src.nrows, src.ncols, src.blk) == (dst.world, dst.nrows, dst.ncols, dst.blk)
    sends: Dict[int, list] = {}
    recvs: Dict[int, list] = {}
    for (i, j) in sorted(src.owned(rank)):
        sends.setdefault(dst.owner(i, j), []).append((src.slot(i, j), dst.slot(i, j)))
    for (i, j) in sorted(dst.owned(rank)):
        recvs.setdefault(src.owner(i, j), []).append(dst.slot(i, j))
    return sends, recvs


def exchange_repartition(slab, src: GridPlan, dst: GridPlan, rank: int):
    """The all-to-all permutation that replaces the reference's ShuffledRDD: every block travels once, untouched, to its owner
    under `dst` (point-to-point, one packed message per peer; CPU tensors over gloo, device tensors over NCCL)."""
    import torch
    import torch.distributed as dist
    out = torch.zeros((dst.local_slots, dst.slot_elems), dtype=slab.dtype, device=slab.device)
    sends, recvs = repartition_routes(src, dst, rank)
    ops, staged, inbox = [], [], []
    for peer, moves in sorted(sends.items()):
        src_idx = torch.tensor([m_[0] for m_ in moves], dtype=torch.long, device=slab.device)
        if peer == rank:
            out[torch.tensor([m_[1] for m_ in moves], dtype=torch.long, device=slab.device)] = slab[src_idx]
        else:
            buf = slab[src_idx].contiguous()
            staged.append(buf)
            ops.append(dist.P2POp(dist.isend, buf, peer))
    for peer, slots in sorted(recvs.items()):
        if peer == rank:
            continue
        buf = torch.empty((len(slots), dst.slot_elems), dtype=slab.dtype, device=slab.device)
        inbox.append((buf, slots))
        ops.append(dist.P2POp(dist.irecv, buf, peer))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for buf, slots in inbox:
        out[torch.tensor(slots, dtype=torch.long, device=slab.device)] = buf
    return out


def sharded_repartition(session, A: ShardedMatrix, dst: GridPlan) -> ShardedMatrix:
    """A on another placement grid of the same ranks (collective)."""
    slab = exchange_repartition(A.slab, A.plan, dst, A.rank)
    esz = slab.element_size()
    ds = session.emptyDataset()
    blocks = dst.owned(A.rank)
    shapes = [dst.block_shape(i, j) for i, j in blocks]
    if blocks:
        ds.put_blocks_device([b[0] for b in blocks], [b[1] for b in blocks], [sh[0] for sh in shapes], [sh[1] for sh in shapes],
                             [slab.data_ptr() + dst.slot(i, j) * dst.slot_elems * esz for i, j in blocks],
                             [1 if A.transposed else 0] * len(blocks))
    return ShardedMatrix(dst, A.rank, slab, ds, session, transposed=A.transposed)


def sharded_elementwise_any(op: str, session, A: ShardedMatrix, B: ShardedMatrix):
    """add / mul / div of two sharded matrices that may live on DIFFERENT placement grids: the right operand is first re-partitioned
    to the left one's grid (MatrixElementAddExecution picks the left partitioner, MatfastExecution.scala:590-606), then the
    co-partitioned kernel runs.  Returns (local result Dataset, keep-alive)."""
    if (B.plan.pr, B.plan.pc) != (A.plan.pr, A.plan.pc):
        B = sharded_repartition(session, B, GridPlan(A.plan.world, B.plan.nrows, B.plan.ncols, B.plan.blk, A.plan.pr, A.plan.pc))
    return sharded_elementwise(op, A, B, A.plan), B


def transpose_plan(plan: GridPlan) -> GridPlan:
    return GridPlan(plan.world, plan.ncols, plan.nrows, plan.blk, plan.pr, plan.pc)


def transpose_routes(plan: GridPlan, rank: int):
    """Block moves of C = A^T on the same grid: block (j, i) of A lives on owner(j, i) = (j % pr, i % pc); as block (i, j) of
    A^T it belongs to (i % pr, j % pc).  Returns (sends, recvs): sends[dst] = [(src_slot, dst_slot)], recvs[src] = [dst_slot],
    both in the same deterministic order (sorted by the A^T block id), so one packed message per peer suffices.
    (The reference's transpose is a flag flip plus a key swap, MatfastExecution.scala:215-236; the re-placement is what its
    next shuffle would do.)"""
    pt = transpose_plan(plan)
    sends: Dict[int, list] = {}
    recvs: Dict[int, list] = {}
    for (j, i) in sorted(plan.owned(rank), key=lambda b: (b[1], b[0])):          # my A blocks, ordered by their A^T id (i, j)
        sends.setdefault(pt.owner(i, j), []).append((plan.slot(j, i), pt.slot(i, j)))
    for (i, j) in sorted(pt.owned(rank)):                                        # the A^T blocks I will own
        recvs.setdefault(plan.owner(j, i), []).append(pt.slot(i, j))
    return sends, recvs


def exchange_transpose(slab, plan: GridPlan, rank: int):
    """Moves the slab's blocks to their owners under the transposed plan (point-to-point, one packed message per peer; works
    on CPU tensors over gloo and on device tensors over NCCL).  Block payloads are not touched: a column-major block (j, i)
    of A IS the row-major block (i, j) of A^T."""
    import torch
    import torch.distributed as dist
    pt = transpose_plan(plan)
    out = torch.zeros((pt.local_slots, pt.slot_elems), dtype=slab.dtype, device=slab.device)
    sends, recvs = transpose_routes(plan, rank)
    ops, staged = [], []
    for dst, moves in sorted(sends.items()):
        src_idx = torch.tensor([m[0] for m in moves], dtype=torch.long, device=slab.device)
        if dst == rank:
            out[torch.tensor([m[1] for m in moves], dtype=torch.long, device=slab.device)] = slab[src_idx]
        else:
            buf = slab[src_idx].contiguous()
            staged.append(buf)
            ops.append(dist.P2POp(dist.isend, buf, dst))
    inbox = []
    for src, slots in sorted(recvs.items()):
        if src == rank:
            continue
        buf = torch.empty((len(slots), pt.slot_elems), dtype=slab.dtype, device=slab.device)
        inbox.append((buf, slots))
        ops.append(dist.P2POp(dist.irecv, buf, src))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for buf, slots in inbox:
        out[torch.tensor(slots, dtype=torch.long, device=slab.device)] = buf
    return out, pt


def sharded_transpose(session, A: ShardedMatrix) -> ShardedMatrix:
    """A^T on the same grid: one packed point-to-point exchange, then the received column-major blocks are registered
    zero-copy as ROW-major blocks of A^T (isTransposed = true) -- no transpose kernel runs, as in the reference."""
    slab, pt = exchange_transpose(A.slab, A.plan, A.rank)
    esz = slab.element_size()
    ds = session.emptyDataset()
    blocks = pt.owned(A.rank)
    shapes = [pt.block_shape(i, j) for i, j in blocks]
    ds.put_blocks_device([b[0] for b in blocks], [b[1] for b in blocks], [sh[0] for sh in shapes], [sh[1] for sh in shapes],
                         [slab.data_ptr() + pt.slot(i, j) * pt.slot_elems * esz for i, j in blocks], [1] * len(blocks))
    return ShardedMatrix(pt, A.rank, slab, ds, A.session, transposed=True)


def sharded_aggregate(kind: str, groups: GridGroups, A: ShardedMatrix):
    """rowSum / colSum / sum / trace of a grid-sharded matrix (RowSum/ColumnSum/Sum/TraceDirectExecution,
    MatfastExecution.scala:239-463): the local reduction kernel per rank, then the reference's reduceByKey(add) across
    partitions becomes one all-reduce of an O(N) vector inside the grid row (rowSum), grid column (colSum) or world
    (sum, trace).  Returns a numpy array: the entries of the rows (rowSum) / columns (colSum) this rank's grid row / column
    owns, in global order, or a scalar."""
    import numpy as np
    import torch
    import torch.distributed as dist
    plan, ds = A.plan, A.dataset
    dev = A.slab.device

    def reduce(vec, group, needed):
        t = torch.from_numpy(vec).to(dev)
        if needed:
            dist.all_reduce(t, group=group)
        return t.cpu().numpy()
    r, c = plan.coords(A.rank)
    if kind == "rowSum":
        loc = {b.rid: b.matrix.to_numpy()[:, 0] for b in ds.rowSum(plan.nrows, plan.ncols).collect()}
        rows = list(range(r, plan.nbr, plan.pr))
        vec = np.concatenate([loc.get(i, np.zeros(plan.block_shape(i, 0)[0])) for i in rows]) if rows else np.zeros(0)
        return reduce(vec, groups.row_group, plan.pc > 1)
    if kind == "colSum":
        loc = {b.cid: b.matrix.to_numpy()[0, :] for b in ds.colSum(plan.nrows, plan.ncols).collect()}
        cols = list(range(c, plan.nbc, plan.pc))
        vec = np.concatenate([loc.get(j, np.zeros(plan.block_shape(0, j)[1])) for j in cols]) if cols else np.zeros(0)
        return reduce(vec, groups.col_group, plan.pr > 1)
    if kind in ("sum", "trace"):
        res = (ds.sum if kind == "sum" else ds.trace)(plan.nrows, plan.ncols).collect()
        v = np.array([res[0].matrix.to_numpy()[0, 0] if res else 0.0])
        return float(reduce(v, None, plan.world > 1)[0])
    raise ValueError(kind)


def bench_main(args, METRIC, UNIT, fp64_peak_tflops, ClockSampler, cpu_reference_sample, int8_peak_tops=None):
    """bench.py's N > 1 arm: one rank per GPU, C-stationary grid, peer pulls overlapped with the multiply."""
    import json
    import time
    import numpy as np
    import torch
    import torch.distributed as dist
    from .dataset import MatfastSession, memcpy_d2h
    from .matrix import DenseMatrix, MatrixBlock

    world = int(os.environ["WORLD_SIZE"])
    rank = int(os.environ["RANK"])
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local_rank)
    dist.init_process_group("nccl", device_id=device)
    n, blk = args.n, args.blk
    nb = n // blk
    plan = GridPlan(world, n, n, blk)
    groups = GridGroups(plan, rank)
    flops = 2.0 * n ** 3
    algo = getattr(args, "algo", 0)

    def allmax(x):
        t = torch.tensor([float(x)], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def allsum(x):
        t = torch.tensor([float(x)], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    stream = torch.cuda.Stream(device=device)
    with torch.cuda.stream(stream):
        s = MatfastSession(device=local_rank, stream=stream.cuda_stream)
        s.set_option("gemm_algo", algo)
        s.set_option("crt_moduli", getattr(args, "crt_moduli", 0))
        A = ShardedMatrix.rand(s, plan, rank, 42, device)
        B = ShardedMatrix.rand(s, plan, rank, 43, device)
        s.sync()
        A.peer_slabs()
        B.peer_slabs()            # collective: CUDA IPC handles exchanged and mapped once
        torch.cuda.synchronize()
        dist.barrier()

        def step():
            return sharded_multiply(s, groups, A, B, plan, plan, nchunks=getattr(args, "pull_chunks", 4))

        def timed(steps):
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(steps):
                out = step()
                del out
            e1.record(stream)
            torch.cuda.synchronize()
            dist.barrier()
            return allmax(e0.elapsed_time(e1) / steps)

        sampler = ClockSampler(local_rank)
        sampler.start()
        for _ in range(args.warmup):
            out = step()
            del out
        torch.cuda.synchronize()
        dist.barrier()
        s.reset_stats()
        sampler.mark()
        ms_max = timed(args.steps)
        clocks = sampler.stop()
        st = s.stats()
        on_tc = st["tc_gemm_launches"] > 0
        launches = allsum(st["kernel_launches"])
        p2p = allsum(st["p2p_bytes"]) / args.steps

        # the dominant kernel alone on this rank (library-side CUDA events), max over ranks
        s.set_option("time_kernels", 1)
        s.reset_stats()
        for _ in range(3):
            out = step()
            del out
        st2 = s.stats()
        s.set_option("time_kernels", 0)
        dpeak, dpeak_src = fp64_peak_tflops()
        if on_tc:
            kern_ms = allmax(st2["tc_gemm_ms_total"] / 3.0)
            ipeak, ipeak_src = int8_peak_tops() if int8_peak_tops else (1979.0, "H100 SXM data sheet, dense INT8")
            ach = st2["tc_int8_ops"] / (kern_ms * 1e-3) / 1e12
            roofline = {"bound": "tensor", "achieved": ach, "peak": ipeak, "unit": "TFLOP/s", "frac": ach / ipeak, "traffic": None,
                        "op": "int8 multiply-add x 2 (TOPS) on wgmma s8, per rank",
                        "kernel": "ozaki2_gemm_2sm_kernel", "kernel_ms": kern_ms,
                        "algorithmic": f"{st2['tc_int8_ops']:.4g} int8 ops per rank per step ({st2['tc_moduli']} moduli x 2 M_loc N_loc K; max-over-ranks kernel time)",
                        "peak_source": ipeak_src,
                        "fp64_equivalent": {"achieved": flops / (ms_max * 1e-3) / 1e12, "dmma_peak": world * dpeak,
                                            "x_dmma_roof": flops / (ms_max * 1e-3) / 1e12 / (world * dpeak)}}
        else:
            kern_ms = allmax(st2["gemm_ms_total"] / 3.0)
            ach = (flops / world) / (kern_ms * 1e-3) / 1e12
            roofline = {"bound": "tensor", "achieved": ach, "peak": dpeak, "unit": "TFLOP/s", "frac": ach / dpeak, "traffic": None,
                        "kernel": "gemm_f64_dmma_kernel<128,128,2,4,5>", "kernel_ms": kern_ms,
                        "algorithmic": f"2*N^3/{world} = {flops / world:.4g} flop per launch per rank (max-over-ranks kernel time)",
                        "peak_source": dpeak_src}

        # ---- correctness of the timed configuration: one output block per rank against numpy fp64 on the host, from the operand
        #      blocks as they sit in the owners' slabs (read through the IPC mappings); MAX over ranks
        def host_reference(i, j):
            from threadpoolctl import threadpool_limits
            pa, pb = A.peer_slabs(), B.peer_slabs()
            want = np.zeros((blk, blk))
            bufa, bufb = np.empty(blk * blk), np.empty(blk * blk)
            with threadpool_limits(limits=8, user_api="blas"):
                for k in range(nb):
                    memcpy_d2h(s, pa[plan.owner(i, k)] + plan.slot(i, k) * plan.slot_elems * 8, bufa)
                    memcpy_d2h(s, pb[plan.owner(k, j)] + plan.slot(k, j) * plan.slot_elems * 8, bufb)
                    want += bufa.reshape(blk, blk).T @ bufb.reshape(blk, blk).T      # blocks are column-major
            return want

        def check_block(dC):
            mine = plan.owned(rank)
            i, j = mine[(len(mine) * 2) // 3]
            got = dC.get_block(i, j).to_numpy()
            want = host_reference(i, j)
            return float(np.max(np.abs(got - want)) / np.max(np.abs(want))), [int(i), int(j)]

        dC, keep = step()
        err, blk_id = check_block(dC)
        nblocks = allsum(len(dC.block_ids()))
        del dC, keep
        check = {"max_rel_err_vs_host_fp64": allmax(err), "blocks_checked": world, "rank0_block": blk_id,
                 "output_blocks_total": int(nblocks), "expected_blocks": nb * nb}

        # ---- the exact native-fp64 kernel (DMMA) on every rank, beside the headline
        dmma = None
        if on_tc:
            try:
                s.set_option("gemm_algo", 1)
                for _ in range(2):
                    out = step()
                    del out
                d_ms = timed(max(3, min(args.steps, 5)))
                dC, keep = step()
                derr, _ = check_block(dC)
                del dC, keep
                dmma = {"algo": "gemm_algo 1: gemm_f64_dmma_kernel on every rank", "value": flops / (d_ms * 1e-3) / 1e9, "unit": UNIT,
                        "ms_per_step": d_ms, "frac_of_dmma_roof": flops / (d_ms * 1e-3) / 1e12 / (world * dpeak),
                        "max_rel_err_vs_host_fp64": allmax(derr)}
            except Exception as e:
                dmma = {"error": str(e)[-200:]}
            finally:
                s.set_option("gemm_algo", algo)
        dist.barrier()

        # ---- end to end: every rank feeds its own A / B blocks from pinned host memory into its slabs, pulls what it needs from
        #      its peers, multiplies, and reads its C blocks back
        hostA = [(k, A.dataset.get_block(*k)) for k in A.dataset.block_ids()]
        hostB = [(k, B.dataset.get_block(*k)) for k in B.dataset.block_ids()]
        pin = lambda v: torch.from_numpy(v).pin_memory().numpy()  # noqa: E731
        pA = [MatrixBlock(i, j, DenseMatrix(m.numRows, m.numCols, pin(m.values), m.isTransposed)) for (i, j), m in hostA]
        pB = [MatrixBlock(i, j, DenseMatrix(m.numRows, m.numCols, pin(m.values), m.isTransposed)) for (i, j), m in hostB]
        ref00 = hostA[0][1].values[:4].copy()
        del hostA, hostB
        outbuf = {k: torch.empty(blk * blk, dtype=torch.float64).pin_memory().numpy() for k in plan.owned(rank)}
        h2d = sum(b.matrix.values.nbytes for b in pA) + sum(b.matrix.values.nbytes for b in pB)
        d2h = sum(v.nbytes for v in outbuf.values())
        eA = ShardedMatrix(plan, rank, torch.zeros_like(A.slab), None, s)
        eB = ShardedMatrix(plan, rank, torch.zeros_like(B.slab), None, s)
        eA.peer_slabs()
        eB.peer_slabs()
        torch.cuda.synchronize()
        dist.barrier()

        side = torch.cuda.Stream(device=device)      # the cross-rank barriers run here, beside the multiply
        nch, chunk_rows, chunk_cols = pull_chunks(plan, plan, rank, getattr(args, "e2e_chunks", 8))
        pA_by_chunk = [[b for b in pA if b.rid in set(rows)] for rows in chunk_rows]
        pB_by_chunk = [[b for b in pB if b.cid in set(cols)] for cols in chunk_cols]
        piece_of_row = {i: ch for ch, rows in enumerate(chunk_rows) for i in rows}
        piece_of_col = {j: ch for ch, cols in enumerate(chunk_cols) for j in cols}
        tick = torch.zeros(1, device=device)

        def gate_after_ingest():
            return ingest_gate(s, side, tick)

        def e2e_step():
            # block rows of A and block columns of B are uploaded alternately, piece by piece (async copies on the ingest stream,
            # one event per block); the multiply is called once and its pulls wait piece by piece for the peers' uploads, so the
            # corner of C that the pieces landed so far unlock is multiplied and read back while the rest is still on the wire
            evs = []
            for ch in range(nch):
                eA.sharded.put_blocks(pA_by_chunk[ch])
                evs.append(gate_after_ingest())
                eB.sharded.put_blocks(pB_by_chunk[ch])
                evs.append(gate_after_ingest())
            dC, keep = sharded_multiply(s, groups, eA, eB, plan, plan, nchunks=nch, gates=[e.cuda_event for e in evs])
            for k in sorted(dC.block_ids(), key=lambda ij: (max(piece_of_row[ij[0]], piece_of_col[ij[1]]), ij)):   # completion order
                dC.get_block(*k, out=outbuf[k])
            stream_barrier(device)             # nobody rewrites a slab while a peer may still be pulling from it
            return dC

        for _ in range(min(2, args.warmup)):
            e2e_step()
        torch.cuda.synchronize()
        dist.barrier()
        # the PCIe floor of the step on this host: the same uploads alone (all ranks at once), nothing else running
        t0 = time.perf_counter()
        for _ in range(2):
            eA.sharded.put_blocks(pA)
            eB.sharded.put_blocks(pB)
            eA.sharded.wait_ingest()       # host-blocking
            eB.sharded.wait_ingest()
        dist.barrier()
        ingest_only_ms = allmax((time.perf_counter() - t0) / 2 * 1e3)
        e2e_steps = max(1, min(args.steps, 5))
        t0 = time.perf_counter()
        for _ in range(e2e_steps):
            e2e_step()
        torch.cuda.synchronize()
        dist.barrier()
        e2e_ms = allmax((time.perf_counter() - t0) / e2e_steps * 1e3)
        dC = e2e_step()
        mine = plan.owned(rank)
        i, j = mine[(len(mine) * 2) // 3]
        e2e_err = float(np.max(np.abs(outbuf[(i, j)].reshape(blk, blk).T - host_reference(i, j))) / np.max(np.abs(outbuf[(i, j)])))
        check["e2e_max_rel_err_vs_host_fp64"] = allmax(e2e_err)
        del dC
        h2d_total, d2h_total = int(allsum(h2d)), int(allsum(d2h))
        torch.cuda.synchronize()
        dist.barrier()
        s.stop()

    if rank == 0:
        line = {
            "metric": METRIC, "value": flops / (ms_max * 1e-3) / 1e9, "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_max, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": f"{n}x{n} fp64 dense multiply, {blk}-block, grid-partitioned {plan.pr}x{plan.pc} over {world}xH100",
                       "parallelism": (f"C-stationary {plan.pr}x{plan.pc} block-cyclic grid; every rank pulls A along its grid row and B along its grid "
                                       "column out of its peers' slabs (CUDA IPC, copy engines over NVLink), chunked and overlapped with the multiply; no reduction"),
                       "inputs": "U(0,1) java.util.Random streams, every block present, column-major",
                       "l2": "per-rank operands after the pulls >> 50 MB L2; no flush needed",
                       "gemm_algo": "auto -> Ozaki-II on wgmma on every rank" if on_tc else "dmma_fp64",
                       "p2p_bytes_per_step": p2p},
            "e2e": {"value": flops / (e2e_ms * 1e-3) / 1e9, "unit": UNIT, "h2d_bytes_per_step": h2d_total,
                    "d2h_bytes_per_step": d2h_total, "ms_per_step": e2e_ms, "steps": e2e_steps,
                    "ingest_only_ms": ingest_only_ms, "pieces": nch,
                    "note": "ingest_only_ms = the step's host->device copies alone on this host (max over ranks): the PCIe floor of the step"},
            "gpu_launches": int(launches), "gpu_launches_per_step_per_rank": st["kernel_launches"] / args.steps,
            "roofline": roofline,
            "clocks": clocks,
            "check": check,
            "dmma_fp64": dmma,
        }
    else:
        line = None
    dist.barrier()
    dist.destroy_process_group()
    return line
