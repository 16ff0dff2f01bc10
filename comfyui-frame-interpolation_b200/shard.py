"""Frame-pair sharding across the GPUs of one box (one process per GPU, torch.distributed for the plumbing).

The per-pair loop of RIFE_VFI.vfi (rife/__init__.py:164-222) is embarrassingly parallel over (pair, timestep)
tasks: task i needs only frames[pair] and frames[pair+1].  Each rank takes a contiguous, task-count-balanced
slice (so skip lists / per-pair multiplier lists stay balanced), uploads only its frame range (one-frame halo)
and the only exchange is the final gather of the interpolated frames on rank 0 (NCCL over NVLink on the GPU box,
gloo in the CPU tests).  Pure host logic: no CUDA here.
"""
from typing import List, Sequence, Tuple

import torch


def shard_tasks(n_tasks: int, world: int) -> List[Tuple[int, int]]:
    """[lo, hi) task slice of every rank: contiguous, sizes differ by at most one, earlier ranks get the extra."""
    base, extra = divmod(n_tasks, world)
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def frame_range(tasks: Sequence[Tuple[int, float]]) -> Tuple[int, int]:
    """[lo, hi) of the source frames a task slice touches (pair p reads frames p and p+1)."""
    if not tasks:
        return (0, 0)
    ps = [p for p, _ in tasks]
    return (min(ps), max(ps) + 2)


def gather_frames(local: torch.Tensor, counts: Sequence[int], dist, dst: int = 0):
    """Variable-size gather of per-rank [n_r, H, W, 3] tensors onto `dst`; returns the concatenation on dst, None
    elsewhere.  Padded to the largest shard so it is a single collective (sizes differ by at most one frame)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    mx = max(counts)
    shape = (mx,) + tuple(local.shape[1:])
    buf = local
    if local.shape[0] != mx:
        buf = torch.zeros(shape, dtype=local.dtype, device=local.device)
        buf[: local.shape[0]] = local
    bufs = [torch.empty(shape, dtype=local.dtype, device=local.device) for _ in range(world)] if rank == dst else None
    dist.gather(buf.contiguous(), bufs, dst=dst)
    if rank != dst:
        return None
    return torch.cat([b[:c] for b, c in zip(bufs, counts)], 0)


def interpolate_sharded(run_tasks, frames: torch.Tensor, tasks: Sequence[Tuple[int, float]], dist, dst: int = 0):
    """Run `run_tasks(frames, task_slice, (frame_lo, frame_hi)) -> [n, H, W, 3]` on this rank's slice and gather.

    `run_tasks` is the engine call on the GPU box (Rife46Engine.interpolate_host / forward) and a stand-in in the
    CPU tests.  Returns all interpolated frames in task order on `dst`."""
    world, rank = dist.get_world_size(), dist.get_rank()
    slices = shard_tasks(len(tasks), world)
    lo, hi = slices[rank]
    mine = list(tasks[lo:hi])
    local = run_tasks(frames, mine, frame_range(mine))
    return gather_frames(local, [b - a for a, b in slices], dist, dst)


def chunk_bounds(n: int, nchunks: int) -> List[Tuple[int, int]]:
    """[lo, hi) row ranges that split n rows into at most nchunks near-equal chunks."""
    nchunks = max(1, min(nchunks, n))
    base, extra = divmod(n, nchunks)
    out, lo = [], 0
    for i in range(nchunks):
        hi = lo + base + (1 if i < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def forward_and_gather(run_slice, local_out: torch.Tensor, counts: Sequence[int], dist, dst: int = 0, nchunks: int = 4,
                       gathered=None):
    """Compute this rank's interpolated frames chunk by chunk and gather every chunk onto `dst` WHILE the next one
    is being computed (the gather of the whole result after the compute would add (world-1) x |result| of inbound
    traffic on dst to every step: 11 GB at world 8 for the 1080p/64-frame workload).

    run_slice(lo, hi) must fill local_out[lo:hi] (asynchronously on the current CUDA stream, or synchronously on
    CPU); local_out has max(counts) rows on every rank (ranks with fewer frames leave the last row unused).  The
    gathers run on a side stream ordered after the chunk's kernels by an event.  Returns the list of per-rank
    [max(counts), ...] buffers on dst (row r of buffer j valid for r < counts[j]), None elsewhere; pass `gathered`
    to reuse the receive buffers between calls."""
    world, rank = dist.get_world_size(), dist.get_rank()
    mx = max(counts)
    assert local_out.shape[0] == mx, "local_out must have max(counts) rows"
    n = counts[rank]
    cuda = local_out.is_cuda
    if rank == dst and gathered is None:
        gathered = [torch.empty_like(local_out) for _ in range(world)]
    comm = torch.cuda.Stream(device=local_out.device) if cuda else None
    for lo, hi in chunk_bounds(mx, nchunks):
        if lo < n:
            run_slice(lo, min(hi, n))
        recv = [g[lo:hi] for g in gathered] if rank == dst else None
        if cuda:
            ev = torch.cuda.Event()
            ev.record()
            comm.wait_event(ev)
            with torch.cuda.stream(comm):
                dist.gather(local_out[lo:hi], recv, dst=dst)
        else:
            dist.gather(local_out[lo:hi].contiguous(), recv, dst=dst)
    if cuda:
        torch.cuda.current_stream(local_out.device).wait_stream(comm)
    return gathered if rank == dst else None


class PushGather:
    """The output-frame gather as copy-engine pushes over NVLink into the destination rank's HBM (GPU box only).

    dist.gather is NCCL send / recv: its kernels need SMs on both ends, and every hot kernel of this path is a persistent
    grid of exactly one CTA per SM - with a few SMs taken by NCCL the last CTAs of each layer wait for a free SM and the
    layer can take up to twice as long.  Here the destination rank allocates one [world, rows, ...]
    buffer, shares it through CUDA IPC, and every rank writes its rows straight into its slice with an ordinary
    device-to-device copy on a side stream (a peer copy = DMA engines over NVLink / NVSwitch, no SMs anywhere), chunk by
    chunk behind the kernels that produce them.  torch.distributed (NCCL) carries the IPC handle once and the barrier that
    ends a step.

    Where the IPC mapping gets no NVLink peer access (some containers) the copy is staged through host memory and is far
    slower than the NCCL gather, so bench.py keeps the NCCL gather (in chunks of one internal pass) and this class is
    opt-in (VFI_GATHER=push) for hosts where IPC peer mappings work."""

    def __init__(self, rows: int, row_shape, dtype, dist, dst: int = 0, device=None):
        import torch.multiprocessing.reductions as red
        self.dist, self.dst = dist, dst
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        box = [None]
        self.buffer = None
        if self.rank == dst:
            self.buffer = torch.empty((self.world, rows) + tuple(row_shape), dtype=dtype, device=self.device)
            fn, args = red.reduce_tensor(self.buffer)
            box = [(fn, args)]
        dist.broadcast_object_list(box, src=dst)
        if self.rank == dst:
            self.remote = self.buffer
        else:
            fn, args = box[0]
            self.remote = fn(*args)      # the destination's buffer, mapped into this process (lives on the dst GPU)
        self.mine = self.remote[self.rank]
        self.stream = torch.cuda.Stream(device=self.device)

    def push(self, local_rows: torch.Tensor, lo: int, hi: int):
        """Copy local_rows[lo:hi] into this rank's slice on the destination, behind the work already queued on the current
        stream (call it right after the kernels that produce these rows)."""
        ev = torch.cuda.Event()
        ev.record()
        self.stream.wait_event(ev)
        with torch.cuda.stream(self.stream):
            self.mine[lo:hi].copy_(local_rows[lo:hi], non_blocking=True)

    def finish(self):
        """All pushes of this rank have landed (the caller still needs a barrier before the destination reads)."""
        torch.cuda.current_stream(self.device).wait_stream(self.stream)

    def close(self):
        self.mine = None
        self.remote = None
        self.buffer = None


def forward_and_push(run_slice, local_out: torch.Tensor, n_rows: int, gather: "PushGather", nchunks: int = 16):
    """Compute this rank's rows chunk by chunk and push every chunk to the destination while the next one computes."""
    for lo, hi in chunk_bounds(n_rows, nchunks):
        run_slice(lo, hi)
        gather.push(local_out, lo, hi)
    gather.finish()


# ------------------------------------------------------------------------------------------------- FILM
def shard_pairs_by_cost(costs: Sequence[float], world: int) -> List[Tuple[int, int]]:
    """Contiguous [lo, hi) pair ranges, one per rank, balancing the summed cost (FILM: a pair costs multiplier - 1
    forward calls, a skipped pair none - film/__init__.py:84-96).  Greedy on the running prefix: rank r ends at the
    first pair where the prefix reaches (r + 1) / world of the total; trailing ranks may get empty ranges."""
    n = len(costs)
    total = float(sum(costs))
    out, lo, acc = [], 0, 0.0
    for r in range(world):
        hi = lo
        if r == world - 1:
            hi = n
        else:
            target = total * (r + 1) / world
            while hi < n and acc + costs[hi] <= target + 1e-9:
                acc += costs[hi]
                hi += 1
            # take the pair that crosses the target if that leaves the split closer to it
            if hi < n and hi < n - (world - 1 - r) + 1 and (target - acc) > (acc + costs[hi] - target):
                acc += costs[hi]
                hi += 1
        out.append((lo, hi))
        lo = hi
    return out


def film_vfi_sharded(run_node, frames: torch.Tensor, multiplier, states, dist, dst: int = 0, device=None):
    """FILM_VFI.vfi over the ranks of one box: frame pairs (with their whole bisection schedules) are independent, so
    every rank runs the node on a contiguous sub-clip (one-frame halo) and the only exchange is the gather of the output
    frames on `dst`.  `run_node(sub_frames, sub_multipliers, sub_states) -> [M_r, H, W, 3]` is the node call
    (`FILM_VFI().vfi(...)[0]`); `states` is None or (frame_indices, is_skip_list).  Returns the full output on `dst`
    (identical to the unsharded node's), None elsewhere."""
    world, rank = dist.get_world_size(), dist.get_rank()
    n = frames.shape[0]
    if isinstance(multiplier, int):
        mults = [multiplier] * (n - 1)
    else:
        mults = list(map(int, multiplier))[: n - 1]
        mults += [2] * (n - 1 - len(mults))

    def skipped(i):
        if states is None:
            return False
        idx, is_skip = states
        return (is_skip and i in idx) or (not is_skip and i not in idx)

    costs = [0.0 if skipped(i) else float(max(mults[i], 1) - 1) + 0.01 for i in range(n - 1)]
    counts_of = lambda lo, hi: sum(0 if skipped(i) else max(mults[i], 1) for i in range(lo, hi))  # noqa: E731
    slices = shard_pairs_by_cost(costs, world)
    lo, hi = slices[rank]
    sub_states = None
    if states is not None:
        # keep-lists must stay keep-lists: list every pair of the sub-clip that is kept / skipped explicitly
        sub_states = ([i - lo for i in range(lo, hi) if skipped(i)], True)
    local = run_node(frames[lo:hi + 1], mults[lo:hi], sub_states)[:-1]  # the trailing frame belongs to the next rank
    counts = [counts_of(a, b) for a, b in slices]
    assert local.shape[0] == counts[rank], (local.shape, counts, rank)
    if device is not None:
        local = local.to(device)
    if local.shape[0] == 0:
        local = torch.zeros((0,) + tuple(frames.shape[1:3]) + (3,), dtype=torch.float32, device=local.device)
    full = gather_frames(local.contiguous(), counts, dist, dst)
    if rank != dst:
        return None
    return torch.cat([full.cpu(), frames[-1:, ..., :3].to(torch.float32)], 0)  # film/__init__.py:104


def generic_vfi_sharded(run_node, frames: torch.Tensor, multiplier: int, states, dist, dst: int = 0, device=None):
    """Nodes that run `generic_frame_loop` (Sepconv VFI, vfi_utils.py:339-389) over the ranks of one box, int multiplier:
    every pair emits its first frame, plus multiplier - 1 new frames unless it is skipped (:260-265, :329-337), and the
    last frame closes the clip - so contiguous pair ranges can run as independent sub-clips and be concatenated.
    `run_node(sub_frames, multiplier, sub_states) -> [M_r, H, W, 3]`.  Returns the full output on `dst`, None elsewhere.
    (List multipliers go through the reference's per-pair quirk - the skip predicate sees index 0 for every pair,
    frame_loop.py - and are not sharded here.)"""
    if not isinstance(multiplier, int):
        raise NotImplementedError("generic_vfi_sharded: int multipliers only")
    world, rank = dist.get_world_size(), dist.get_rank()
    n = frames.shape[0]

    def skipped(i):
        if states is None:
            return False
        idx, is_skip = states
        return (is_skip and i in idx) or (not is_skip and i not in idx)

    costs = [0.01 if skipped(i) else float(multiplier - 1) + 0.01 for i in range(n - 1)]
    slices = shard_pairs_by_cost(costs, world)
    counts = [sum(1 if skipped(i) else multiplier for i in range(a, b)) for a, b in slices]
    lo, hi = slices[rank]
    if hi > lo:
        sub_states = None if states is None else ([i - lo for i in range(lo, hi) if skipped(i)], True)
        local = run_node(frames[lo:hi + 1], multiplier, sub_states)[:-1]
    else:
        local = torch.zeros((0,) + tuple(frames.shape[1:3]) + (3,), dtype=torch.float32)
    assert local.shape[0] == counts[rank], (local.shape, counts, rank)
    if device is not None:
        local = local.to(device)
    full = gather_frames(local.contiguous(), counts, dist, dst)
    if rank != dst:
        return None
    return torch.cat([full.cpu(), frames[-1:, ..., :3].to(torch.float32)], 0)
