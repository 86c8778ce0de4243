"""Instance-level data parallelism (SURVEY.md §8e): simulator instances are independent (own seed, own RNG,
own nodes — simulator.rs:200-250), so the batch is sharded contiguously over ranks with NO data-path
collective; one all-gather of the per-instance summaries ``{commit_count[N], state_key[N], rounds}`` happens at
the end of a run.  One process per GPU, ``torch.distributed`` (NCCL over NVLink/NVSwitch between H100s, gloo in
the CPU tests).

``ShardedBatchSimulator`` is the product's multi-GPU entry: it owns the sharding (``shard_bounds``), this rank's
``BatchSimulator`` handle and the all-gather.  With NCCL the gather reads the library's device-resident result
buffers in place (``lbft_device_buffer``): no host round trip.  (One host thread driving several GPUs without
``torch.distributed`` is the other route: ``lbft_run_async`` / ``lbft_wait`` on one handle per device, see
``tests/cabi/multi_handle.c`` and ``bft-lib-gpu``.)"""
import numpy as np


def shard_bounds(total, world, rank):
    """GPU g gets instances [g*I/G, (g+1)*I/G)."""
    return (rank * total) // world, ((rank + 1) * total) // world


def all_gather_rows(local, world, dist=None):
    """All-gather equally-shaped per-rank tensors along dim 0 (device tensors for NCCL, CPU for gloo)."""
    import torch
    if world == 1 or dist is None:
        return local
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous())
    return out


class _DeviceView:
    """``__cuda_array_interface__`` over a library-owned device buffer (no copy)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}


class ShardedResult:
    """Whole-job summaries after the all-gather, plus this rank's own ``BatchResult`` (``.local``).  ``block`` is the gathered
    ``[world, bytes]`` tensor (device memory with NCCL): per rank the last states [I][N] u64, commit counts [I][N] u32 and
    active rounds [I] u32 of its shard; it is decoded on the host on first access."""

    def __init__(self, local, block, instances_per_rank, num_nodes, lo, hi):
        self.local, self.block, self.lo, self.hi = local, block, lo, hi
        self._shape, self._decoded = (instances_per_rank, num_nodes), None

    def _decode(self):
        if self._decoded is None and self.block is None:  # one rank: the whole job is this rank's shard
            self._decoded = (self.local.commit_counts, self.local.last_committed_states, self.local.active_rounds)
        if self._decoded is None:
            I, N = self._shape
            b = self.block.detach().cpu().numpy() if hasattr(self.block, "detach") else np.asarray(self.block)
            b = np.ascontiguousarray(b).reshape(-1, I * N * 12 + I * 4)
            ns, nc = I * N * 8, I * N * 4
            self._decoded = (np.ascontiguousarray(b[:, ns:ns + nc]).view(np.uint32).reshape(-1, N),
                             np.ascontiguousarray(b[:, :ns]).view(np.uint64).reshape(-1, N),
                             np.ascontiguousarray(b[:, ns + nc:]).view(np.uint32).reshape(-1))
        return self._decoded

    @property
    def commit_counts(self):
        """[all instances, node] ``committed_history().len()``"""
        return self._decode()[0]

    @property
    def last_committed_states(self):
        return self._decode()[1]

    @property
    def active_rounds(self):
        return self._decode()[2]


class ShardedBatchSimulator:
    """The batch of ``seeds`` (the WHOLE job's, identical on every rank) spread over ``world`` ranks.

    ``make_local(seeds_shard)`` builds this rank's simulator (default: a ``BatchSimulator`` on ``device``); the CPU
    tests inject a host stand-in with the same ``create / set_seeds / run`` surface, so the sharding and gathering
    logic is covered without a GPU."""

    def __init__(self, seeds, num_nodes, *args, rank=0, world=1, dist=None, device=0, make_local=None, **kw):
        seeds = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
        if len(seeds) % world != 0:
            raise ValueError("number of instances (%d) must be a multiple of the world size (%d): the summaries travel in one "
                             "all_gather_into_tensor" % (len(seeds), world))
        self.total, self.num_nodes, self.rank, self.world, self.dist, self.device = len(seeds), int(num_nodes), rank, world, dist, device
        self.lo, self.hi = shard_bounds(self.total, world, rank)
        if make_local is None:
            from .simulator import BatchSimulator

            def make_local(shard):
                return BatchSimulator(shard, num_nodes, *args, device=device, **kw)
        self.local = make_local(seeds[self.lo:self.hi])
        self._views = None

    def create(self, max_clock):
        self.local.create(int(max_clock))
        self._views = None
        return self

    def close(self):
        self.local.close()

    def set_seeds(self, seeds):
        """Re-seed the whole job; this rank keeps its contiguous shard."""
        seeds = np.ascontiguousarray(np.asarray(seeds, dtype=np.uint64).reshape(-1))
        if len(seeds) != self.total:
            raise ValueError("expected %d seeds" % self.total)
        self.local.set_seeds(seeds[self.lo:self.hi])

    # -- the one collective of the path ---------------------------------------------------------------
    def _device_summary(self):
        """Torch view of the library's device-resident summary block of this shard: last states [I][N] u64, commit counts
        [I][N] u32, active rounds [I] u32, contiguous (``lbft_device_buffer(5)``) — NCCL gathers it in place."""
        import torch
        if self._views is None:
            ptr, nbytes = self.local.device_buffer(5)
            self._views = torch.as_tensor(_DeviceView(ptr, (nbytes,), "|u1"), device="cuda:%d" % self.device)
        return self._views

    def gather(self, local_result=None):
        """ONE all-gather of ``{state_key[N], commit_count[N], rounds}`` of every rank's shard (SURVEY §8e), complete when it
        returns.  On a CUDA backend the source is the device-resident summary block; otherwise the host arrays of
        ``local_result`` packed the same way.  Returns the gathered ``[world, bytes]`` block (see ``ShardedResult``)."""
        import torch
        if self.world == 1 or self.dist is None:
            return None  # nothing to gather: ShardedResult reads this rank's arrays
        on_device = self._gathers_on_device()
        if on_device:
            block = self._device_summary()
        else:
            block = torch.as_tensor(np.concatenate([
                np.ascontiguousarray(local_result.last_committed_states, dtype=np.uint64).reshape(-1).view(np.uint8),
                np.ascontiguousarray(local_result.commit_counts, dtype=np.uint32).reshape(-1).view(np.uint8),
                np.ascontiguousarray(local_result.active_rounds, dtype=np.uint32).reshape(-1).view(np.uint8)]))
        allb = all_gather_rows(block.reshape(1, -1), self.world, self.dist if self.world > 1 else None)
        if on_device:
            torch.cuda.current_stream(allb.device).synchronize()  # the results are complete (and the sources free) on return
        return allb

    def _gathers_on_device(self):
        return self.dist is not None and self.world > 1 and self.dist.get_backend() == "nccl"

    def run(self, strict=True):
        """``lbft_run`` on this rank's shard (host seeds in, host summaries out) + the all-gather."""
        res = self.local.run(strict=strict)
        return ShardedResult(res, self.gather(res), self.hi - self.lo, self.num_nodes, self.lo, self.hi)

    def run_stream(self, batches, strict=True):
        """A sequence of whole-job seed batches with one run always in flight on every rank (``lbft_run_async`` /
        ``lbft_wait``): yields one ``ShardedResult`` per batch, in order.  While batch k runs, batch k + 1 is staged in the
        other pinned seed buffer; when batch k's summaries have landed, its all-gather reads the device buffers, batch k + 1
        is launched, and only then are batch k's summaries copied into the caller's arrays — the host side of a step
        overlaps the next kernel.  Local runners without ``run_async`` (the CPU stand-ins of the tests) run one by one."""
        if not hasattr(self.local, "run_async"):
            for seeds in batches:
                self.set_seeds(seeds)
                yield self.run(strict=strict)
            return
        it = iter(batches)
        first = next(it, None)
        if first is None:
            return
        n, on_device = self.hi - self.lo, self._gathers_on_device()
        box = {}

        def gather_device():
            box["block"] = self.gather()

        self.set_seeds(first)
        self.local.run_async()
        inflight = True
        try:
            nxt = next(it, None)
            while True:
                if nxt is not None:
                    self.set_seeds(nxt)
                inflight = False
                res = self.local.wait(strict=strict, relaunch=nxt is not None, before_relaunch=gather_device if on_device else None)
                inflight = nxt is not None
                block = box.pop("block", None) if on_device else self.gather(res)
                yield ShardedResult(res, block, n, self.num_nodes, self.lo, self.hi)
                if nxt is None:
                    return
                nxt = next(it, None)
        finally:
            if inflight and hasattr(self.local, "drain"):  # the consumer stopped early: leave the handle idle
                self.local.drain()

    def loop_until(self, max_clock, strict=True):
        """``Simulator::new`` + ``loop_until(max_clock)`` for the whole job (simulator.rs:200-250, 380-475)."""
        self.create(max_clock)
        return self.run(strict=strict)


def run_sharded(seeds, num_nodes, max_clock, rank, world, run_local, dist=None, device=None):
    """Functional form kept for callers that bring their own local runner: ``run_local(seeds_shard) -> (commit_counts[I_r,N],
    last_states[I_r,N])``; returns the whole job's two arrays on every rank."""
    class _Local:
        def __init__(self, shard):
            self.shard = shard

        def create(self, max_clock):
            return self

        def close(self):
            pass

        def set_seeds(self, shard):
            self.shard = shard

        def run(self, strict=True):
            counts, states = run_local(self.shard)
            return type("R", (), {"commit_counts": np.asarray(counts, dtype=np.uint32), "last_committed_states": np.asarray(states, dtype=np.uint64),
                                  "active_rounds": np.zeros(len(self.shard), dtype=np.uint32)})()

    sim = ShardedBatchSimulator(seeds, num_nodes, rank=rank, world=world, dist=dist, make_local=_Local)
    res = sim.loop_until(max_clock)
    total = len(np.asarray(seeds).reshape(-1))
    return res.commit_counts.reshape(total, num_nodes), res.last_committed_states.reshape(total, num_nodes)
