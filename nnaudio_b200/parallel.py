"""Batch-sharded multi-GPU execution (SURVEY.md §8e).

Clips are independent, so the transform itself needs no collective: rank ``r``
(one process per GPU, ``torch.distributed``/NCCL) owns a contiguous slice of the
batch.  The only exchange is the optional gather of the output spectrograms,
one ``all_gather_into_tensor`` over NVLink/NVSwitch (the batch is the outermost
output dimension, so shards are contiguous blocks of the gathered tensor).

The reference's counterpart is ``torch.nn.DataParallel`` (single process,
scatter → replicate the module every forward → gather; tests/test_stft.py:122-141).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(total: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous balanced partition of ``total`` clips over ``world`` ranks
    (the first ``total % world`` ranks hold one extra clip)."""
    base, extra = divmod(total, world)
    bounds, start = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        bounds.append((start, start + n))
        start += n
    return bounds


class BatchShardedTransform:
    """Wrap a spectrogram module (or any ``x -> y`` callable whose leading
    dimension is the clip axis) for one-process-per-GPU execution.

    ``forward(x_local)`` transforms this rank's shard and, when ``gather`` is
    true, returns the spectrograms of the WHOLE batch on every rank.
    """

    def __init__(self, transform: Callable[[torch.Tensor], torch.Tensor],
                 group: Optional[dist.ProcessGroup] = None, gather: bool = True,
                 reserve_sms: int = 8):
        """``reserve_sms``: SMs kept out of the persistent tensor-core grids while a
        gather may be in flight — the kernels otherwise occupy every SM and NCCL's
        CTAs could only start at their tail (no overlap)."""
        self.transform = transform
        self.group = group
        self.gather = gather
        if gather and dist.is_initialized() and dist.get_world_size(group) > 1 and reserve_sms > 0:
            try:
                from . import _C
                _C.set_sm_reserve(reserve_sms)
            except Exception:  # noqa: BLE001  (CPU-only test processes have no use for it)
                pass
        self._buf = None
        self._slots = {}

    @property
    def world(self) -> int:
        return dist.get_world_size(self.group) if dist.is_initialized() else 1

    @property
    def rank(self) -> int:
        return dist.get_rank(self.group) if dist.is_initialized() else 0

    def local_slice(self, x_global: torch.Tensor) -> torch.Tensor:
        """This rank's shard of a batch that every rank holds (or can index)."""
        lo, hi = shard_bounds(x_global.shape[0], self.world)[self.rank]
        return x_global[lo:hi]

    def __call__(self, x_local: torch.Tensor, total: Optional[int] = None) -> torch.Tensor:
        return self.forward(x_local, total)

    def forward(self, x_local: torch.Tensor, total: Optional[int] = None) -> torch.Tensor:
        y = self.transform(x_local)
        world = self.world
        if not self.gather or world == 1:
            return y
        n_local = y.shape[0]
        if total is None:
            total = n_local * world  # equal shards
        bounds = shard_bounds(total, world)
        n_max = max(hi - lo for lo, hi in bounds)
        if (n_local, ) != (bounds[self.rank][1] - bounds[self.rank][0], ):
            raise ValueError(f"rank {self.rank}: local batch {n_local} does not match its shard {bounds[self.rank]}")
        y = y.contiguous()
        if n_local < n_max:  # ragged tail: pad to the common shard size for the collective
            pad = torch.zeros((n_max - n_local,) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
            y = torch.cat((y, pad), 0)
        shape = (world * n_max,) + tuple(y.shape[1:])
        if self._buf is None or self._buf.shape != shape or self._buf.device != y.device:
            self._buf = torch.empty(shape, dtype=y.dtype, device=y.device)
        dist.all_gather_into_tensor(self._buf, y, group=self.group)
        if n_max * world == total:
            return self._buf
        parts = [self._buf[r * n_max: r * n_max + (hi - lo)] for r, (lo, hi) in enumerate(bounds)]
        return torch.cat(parts, 0)

    # ------------------------------------------------------------------ #
    # Gather without NCCL kernels and without SMs (SURVEY.md 8(e) fusion target, first step).  Every
    # rank owns a symmetric-memory buffer holding the WHOLE gathered output (two rotating slots);
    # after its transform a rank pushes its shard into the same slice of every peer's buffer
    # (``gather_to='all'``) or of the root's only (``gather_to='root'``: what the north star names;
    # 1/world of the fabric bytes) with plain device-to-device copies over NVLink -- copy engines,
    # so the persistent kernels keep every SM and nothing is reserved for a collective.  Two
    # device-side barriers per step order the slot reuse (every rank has consumed the slot) and the
    # arrival of the pushes.
    def _symm_setup(self, y: torch.Tensor):
        import torch.distributed._symmetric_memory as symm_mem

        world = self.world
        shape = (2, world * y.shape[0]) + tuple(y.shape[1:])
        if getattr(self, "_symm_shape", None) != (shape, y.dtype, y.device):
            group = self.group if self.group is not None else dist.group.WORLD
            buf = symm_mem.empty(shape, dtype=y.dtype, device=y.device)
            hdl = symm_mem.rendezvous(buf, group)
            self._symm = (buf, hdl, [hdl.get_buffer(r, shape, y.dtype) for r in range(world)])
            self._symm_streams = [torch.cuda.Stream(y.device) for _ in range(2)]
            self._symm_consumed = [None, None]
            self._symm_shape = (shape, y.dtype, y.device)
        return self._symm

    class _SymmWork:
        def __init__(self, event):
            self.event = event

        def wait(self):
            """Make the current stream wait for the gathered slot."""
            torch.cuda.current_stream().wait_event(self.event)
            return True

    def release(self, slot: int):
        """Record that the consumer is finished with ``slot`` (call after the last kernel that reads
        the gathered tensor has been enqueued on the current stream).  No-op for the NCCL path."""
        if getattr(self, "_symm_consumed", None) is None:
            return
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self._symm_consumed[slot] = ev

    def forward_async_symm(self, x_local: torch.Tensor, slot: int = 0, gather_to: str = "all",
                           root: int = 0):
        """Like :meth:`forward_async` with the copy-engine gather described above.  Returns
        ``(work, gathered)``; call ``work.wait()`` before reading ``gathered`` and
        ``self.release(slot)`` when done with it.  With ``gather_to='root'`` only rank ``root``'s
        ``gathered`` holds the other ranks' shards."""
        y = self.transform(x_local).contiguous()
        world = self.world
        if not self.gather or world == 1:
            return None, y
        buf, hdl, peers = self._symm_setup(y)
        n = y.shape[0]
        lo = self.rank * n
        cur = torch.cuda.current_stream(y.device)
        ev_y = torch.cuda.Event()
        ev_y.record(cur)
        s, s2 = self._symm_streams
        with torch.cuda.stream(s):
            s.wait_event(ev_y)
            if self._symm_consumed[slot] is not None:
                s.wait_event(self._symm_consumed[slot])
            hdl.barrier(channel=2 * slot)          # every rank is done reading this slot
            if gather_to == "root":
                peers[root][slot, lo:lo + n].copy_(y, non_blocking=True)
            else:
                # two copy streams: two DMA engines drive the NVLink ports together
                ev_b = torch.cuda.Event()
                ev_b.record(s)
                s2.wait_event(ev_b)
                for i in range(world):
                    st = s if (i & 1) == 0 else s2
                    with torch.cuda.stream(st):
                        peers[(self.rank + i) % world][slot, lo:lo + n].copy_(y, non_blocking=True)
                ev_2 = torch.cuda.Event()
                ev_2.record(s2)
                s.wait_event(ev_2)
            hdl.barrier(channel=2 * slot + 1)      # every rank's pushes into this slot have landed
            ev_done = torch.cuda.Event()
            ev_done.record(s)
        y.record_stream(s)
        y.record_stream(s2)
        return BatchShardedTransform._SymmWork(ev_done), buf[slot]

    # ------------------------------------------------------------------ #
    # Gather with NO kernels at all (round 2 default): the transform writes its shard straight into
    # its slice of a symmetric-memory buffer (``_C.output_into``), copy engines push the slice over
    # NVLink into the same slice of every destination's buffer, and the slot handshakes are stream
    # memory operations (cuStreamWriteValue32 / cuStreamWaitValue32 on flag words in symmetric
    # memory): a torch barrier KERNEL or a local staging copy would have to squeeze onto SMs the
    # transform occupies (tools/symm_diag.py measures both next to the persistent kernels).
    #   flags[slot][0][r] on rank d: "rank r's shard of use #c has landed in d's slot"   (r writes it)
    #   flags[slot][1][d] on rank r: "rank d has consumed use #c of the slot"             (d writes it)
    def _peer_setup(self, shard_shape, dtype, device):
        import torch.distributed._symmetric_memory as symm_mem

        world = self.world
        shape = (2, world * shard_shape[0]) + tuple(shard_shape[1:])
        key = (shape, dtype, device)
        if getattr(self, "_peer_key", None) != key:
            group = self.group if self.group is not None else dist.group.WORLD
            buf = symm_mem.empty(shape, dtype=dtype, device=device)
            hdl = symm_mem.rendezvous(buf, group)
            flags = symm_mem.empty((2, 2, world), dtype=torch.int32, device=device)
            flags.zero_()
            torch.cuda.synchronize(device)
            fh = symm_mem.rendezvous(flags, group)
            dist.barrier(group=self.group)  # every rank's flags are zero before anybody signals
            self._peer = dict(
                buf=buf, flags=flags,
                bufs=[hdl.get_buffer(r, shape, dtype) for r in range(world)],
                flag_ptr=[fh.get_buffer(r, (2, 2, world), torch.int32).data_ptr() for r in range(world)],
                streams=[torch.cuda.Stream(device) for _ in range(4)],
                use=[0, 0], pushed=[None, None], handles=(hdl, fh))
            self._peer_key = key
        return self._peer

    class _PeerWork:
        def __init__(self, owner, slot, use, sources):
            self.owner, self.slot, self.use, self.sources = owner, slot, use, sources

        def wait(self):
            """Make the current stream wait until every source's shard of this use has landed."""
            from . import _C
            st = self.owner._peer
            cur = torch.cuda.current_stream()
            me, world = self.owner.rank, self.owner.world
            for r in self.sources:
                if r != me:
                    addr = st["flag_ptr"][me] + 4 * ((self.slot * 2 + 0) * world + r)
                    _C.stream_wait_value32_geq(cur, addr, self.use)
            if st["pushed"][self.slot] is not None:
                cur.wait_event(st["pushed"][self.slot])
            return True

    def release_peer(self, slot: int, dests=None):
        """The consumer is finished with ``slot``: tell every source (stream-ordered after the work
        queued on the current stream)."""
        from . import _C
        st = self._peer
        cur = torch.cuda.current_stream()
        me, world = self.rank, self.world
        if dests is not None and me not in dests:
            return
        for r in range(world):
            if r != me:
                addr = st["flag_ptr"][r] + 4 * ((slot * 2 + 1) * world + me)
                _C.stream_write_value32(cur, addr, st["use"][slot])

    def forward_async_peer(self, x_local: torch.Tensor, slot: int = 0, gather_to: str = "root",
                           root: int = 0):
        """Transform this rank's shard directly into the gather buffer and push it to the
        destinations (``gather_to``: 'root' = rank ``root`` only, 'all' = every rank).  Returns
        ``(work, gathered)``: ``work.wait()`` before reading ``gathered`` on a destination,
        ``release_peer(slot)`` when done with it."""
        from . import _C
        world, me = self.world, self.rank
        if not self.gather or world == 1:
            return None, self.transform(x_local)
        dests = list(range(world)) if gather_to == "all" else [root]
        st = getattr(self, "_peer", None)
        if st is None:
            y0 = self.transform(x_local)      # first call: learn the output shape
            st = self._peer_setup(tuple(y0.shape), y0.dtype, y0.device)
            del y0
        n = st["buf"].shape[1] // world
        lo = me * n
        mine = st["buf"][slot, lo:lo + n]
        cur = torch.cuda.current_stream(x_local.device)
        if st["pushed"][slot] is not None:
            cur.wait_event(st["pushed"][slot])   # my previous pushes out of this slice are done
        st["use"][slot] += 1
        use = st["use"][slot]
        if me in dests and use > 1:
            pass  # my own consumer's release is stream-ordered on `cur` already
        with _C.output_into(mine):
            y = self.transform(x_local)
        if y.data_ptr() != mine.data_ptr():
            mine.copy_(y)                        # a transform that did not take the buffer
        ev_y = torch.cuda.Event()
        ev_y.record(cur)
        targets = [d for d in dests if d != me]
        if targets:
            streams = st["streams"]
            # several copy engines per push: a shard goes out as row chunks on different streams
            # (one destination: 4 chunks; many destinations: the destinations themselves spread over
            # the streams)
            n_chunks = max(1, min(len(streams) // len(targets), n))
            jobs = []
            for d in targets:
                for c in range(n_chunks):
                    r0, r1 = lo + (n * c) // n_chunks, lo + (n * (c + 1)) // n_chunks
                    jobs.append((d, r0, r1, c == n_chunks - 1))
            used = set()
            pending = {d: [] for d in targets}
            for i, (d, r0, r1, last) in enumerate(jobs):
                s = streams[i % len(streams)]
                with torch.cuda.stream(s):
                    if id(s) not in used:
                        s.wait_event(ev_y)
                        used.add(id(s))
                    # destination d has consumed the previous use of this slot
                    _C.stream_wait_value32_geq(
                        s, st["flag_ptr"][me] + 4 * ((slot * 2 + 1) * world + d), use - 1)
                    st["bufs"][d][slot, r0:r1].copy_(st["buf"][slot, r0:r1], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(s)
                    pending[d].append(ev)
            # "landed" flag of destination d: after ALL of its chunks (any stream)
            s0 = streams[0]
            with torch.cuda.stream(s0):
                for d in targets:
                    for ev in pending[d]:
                        s0.wait_event(ev)
                    _C.stream_write_value32(
                        s0, st["flag_ptr"][d] + 4 * ((slot * 2 + 0) * world + me), use)
                done = torch.cuda.Event()
                done.record(s0)
            st["pushed"][slot] = done
        sources = list(range(world)) if me in dests else []
        return BatchShardedTransform._PeerWork(self, slot, use, sources), st["buf"][slot]

    def forward_async(self, x_local: torch.Tensor, slot: int = 0):
        """Pipelined variant for back-to-back batches with equal shards: transform
        the shard, enqueue the output all-gather on NCCL's stream and return
        ``(work, gathered)`` immediately.  ``work.wait()`` makes the CURRENT stream
        wait for the gather; until then the next batch's transform overlaps it.
        ``slot`` selects one of the caller's rotating gather buffers."""
        y = self.transform(x_local).contiguous()
        world = self.world
        if not self.gather or world == 1:
            return None, y
        shape = (world * y.shape[0],) + tuple(y.shape[1:])
        buf = self._slots.get(slot)
        if buf is None or buf.shape != shape or buf.device != y.device:
            buf = torch.empty(shape, dtype=y.dtype, device=y.device)
            self._slots[slot] = buf
        work = dist.all_gather_into_tensor(buf, y, group=self.group, async_op=True)
        return work, buf
