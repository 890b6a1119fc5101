"""Batch sharding across GPUs (SURVEY.md §8e): one process per GPU, contiguous split of dim 0, no
data-path collective.  The only exchange on the path is an all-gather of the per-item loudness vector
(``[B/W] f32`` per rank -> ``[B]``), for whole-batch loudness statistics / logging; with NCCL it is issued
on a side stream so that it overlaps the spectral kernel.  Works with any ``torch.distributed`` backend
(NCCL over NVLink between the GPUs of one node, gloo in the CPU tests)."""
from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(batch_size: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Items ``[lo, hi)`` owned by ``rank``: contiguous, sizes differ by at most one, in rank order."""
    base, rem = divmod(batch_size, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(x, rank: Optional[int] = None, world_size: Optional[int] = None):
    """Slice a ``[B, ...]`` tensor or an ``AudioSignal`` along the batch dim for this rank."""
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_initialized() else 1
    n = x.batch_size if hasattr(x, "batch_size") else x.shape[0]
    lo, hi = shard_bounds(n, rank, world_size)
    return x[lo:hi]


class LoudnessGather:
    """All-gather of per-item loudness across ranks, optionally on a CUDA side stream."""

    def __init__(self, group=None, side_stream: Optional["torch.cuda.Stream"] = None):
        self.group = group
        self.side = side_stream
        self._out = None

    def __call__(self, loud_local: torch.Tensor, counts=None) -> torch.Tensor:
        """``loud_local`` [B_local] -> [B_total] (equal shard sizes, or ``counts`` per rank)."""
        if not dist.is_initialized() or dist.get_world_size(self.group) == 1:
            return loud_local
        world = dist.get_world_size(self.group)
        if counts is None or len(set(counts)) == 1:
            out = torch.empty(world * loud_local.numel(), dtype=loud_local.dtype, device=loud_local.device)
            if self.side is not None and loud_local.is_cuda:
                self.side.wait_stream(torch.cuda.current_stream(loud_local.device))
                with torch.cuda.stream(self.side):
                    dist.all_gather_into_tensor(out, loud_local.contiguous(), group=self.group)
                loud_local.record_stream(self.side)
            else:
                dist.all_gather_into_tensor(out, loud_local.contiguous(), group=self.group)
            return out
        # uneven shards: pad to the largest, gather, drop the padding (all_gather needs equal sizes)
        cmax = max(counts)
        padded = torch.zeros(cmax, dtype=loud_local.dtype, device=loud_local.device)
        padded[: loud_local.numel()] = loud_local
        out = torch.empty(world * cmax, dtype=loud_local.dtype, device=loud_local.device)
        dist.all_gather_into_tensor(out, padded, group=self.group)
        return torch.cat([out[r * cmax: r * cmax + c] for r, c in enumerate(counts)])

    def wait(self):
        """Make the current stream wait for a side-stream gather before its result is consumed."""
        if self.side is not None:
            torch.cuda.current_stream().wait_stream(self.side)


class PeerLoudnessExchange:
    """One-sided exchange of the per-item loudness vector over NVLink peer memory (``csrc/peer.cu``): every rank
    stores its ``[n]`` floats into a small cudaIpc-mapped buffer of every peer and publishes a sequence number.
    No rendezvous and no NCCL kernel; ``torch.distributed`` (any backend) is used once, to swap the 64-byte IPC
    handles.  All ranks must live on one node.

    The statistic is logging data, so NOTHING here can stall the data path: every kernel of the exchange is issued
    on the exchange's own side stream (ordered after the producer of the vector by an event), ``put`` and ``latest``
    never wait for another rank, and only ``collect`` -- the lock-step form, for validation and exact-step
    statistics -- spins (bounded), still on the side stream.

    Per step:  ``seq = ex.put(loud_local)``; whenever statistics are wanted ``vals, seqs = ex.latest()``
    (``[world, n]`` newest complete vector of every rank and the sequence number each row carries).  Slots rotate
    over four sequence numbers and are seqlock-protected, so no ordering between puts and reads is required.
    """

    def __init__(self, n_max: int, device=None, group=None, lib=None):
        import ctypes

        from . import _lib

        assert dist.is_initialized(), "PeerLoudnessExchange needs torch.distributed (for the handle swap only)"
        self.lib = lib if lib is not None else _lib.get_lib()
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.n_max = int(n_max)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else "cpu"
        self.device = torch.device(device)  # "cpu" only with the CPU-simulated library (set-up protocol tests)
        self._ct = ctypes
        # Set-up is all-or-nothing ACROSS ranks: every rank takes part in both handle/status exchanges whatever
        # happened locally, so a failure anywhere (no cudaIpc in this container, a rank on another node, ...) makes
        # every rank raise together and the caller can fall back consistently instead of dead-locking.
        self.local, self._opened, err = None, [], None
        self.peers = (ctypes.c_void_p * self.world)()
        handle = None
        import contextlib

        with (torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext()):
            try:
                ptr = ctypes.c_void_p()
                hbuf = (ctypes.c_ubyte * 64)()
                self.lib.check(self.lib.b2a_peer_buffer_create(self.world, self.n_max, ctypes.byref(ptr), hbuf))
                self.local, handle = ptr.value, bytes(hbuf)
            except Exception as e:  # noqa: BLE001
                err = f"rank {self.rank}: {e}"
            handles = [None] * self.world
            dist.all_gather_object(handles, handle, group=group)
            if err is None and all(h is not None for h in handles):
                try:
                    for r, h in enumerate(handles):
                        if r == self.rank:
                            self.peers[r] = self.local
                            continue
                        p = ctypes.c_void_p()
                        buf = (ctypes.c_ubyte * 64).from_buffer_copy(h)
                        self.lib.check(self.lib.b2a_peer_buffer_open(buf, ctypes.byref(p)))
                        self.peers[r] = p.value
                        self._opened.append(p.value)
                except Exception as e:  # noqa: BLE001
                    err = f"rank {self.rank}: {e}"
            elif err is None:
                err = "a peer could not create its buffer"
            errs = [None] * self.world
            dist.all_gather_object(errs, err, group=group)
            if any(e is not None for e in errs):
                for p in self._opened:
                    self.lib.b2a_peer_buffer_close(ctypes.c_void_p(p))
                if self.local is not None:
                    self.lib.b2a_peer_buffer_destroy(ctypes.c_void_p(self.local))
                self.local = None
                raise RuntimeError("peer exchange unavailable: " + "; ".join(e for e in errs if e))
        dist.barrier(group=group)  # every rank has mapped every buffer before the first put
        self.seq = 0
        self._n = {}
        self.launches = 0  # kernels launched by put / latest / collect
        self.side = torch.cuda.Stream(device=self.device) if self.device.type == "cuda" else None
        self._ev = torch.cuda.Event() if self.side is not None else None

    def _on_side(self, producer_stream=None):
        """Context that makes the side stream current, ordered after everything enqueued so far on the producer's
        stream (the caller's current stream by default)."""
        import contextlib

        if self.side is None:
            return contextlib.nullcontext()
        cur = producer_stream if producer_stream is not None else torch.cuda.current_stream(self.device)
        self._ev.record(cur)
        self.side.wait_event(self._ev)
        return torch.cuda.stream(self.side)

    def _stream_ptr(self):
        return self._ct.c_void_p(self.side.cuda_stream if self.side is not None else 0)

    def put(self, loud_local: torch.Tensor) -> int:
        """Publish this rank's vector as the next sequence number (side stream, never waits); returns the number."""
        assert loud_local.dtype == torch.float32 and loud_local.is_contiguous()
        assert loud_local.device.type == self.device.type
        n = loud_local.numel()
        assert 1 <= n <= self.n_max
        self.seq += 1
        self._n[self.seq] = n
        while len(self._n) > 8:
            self._n.pop(min(self._n))
        with self._on_side():
            self.launches += self.lib.call(self.lib.b2a_peer_put_f32, self._ct.c_void_p(loud_local.data_ptr()), n,
                                           self.peers, self.world, self.rank, self.n_max, self.seq, self._stream_ptr())
        if self.side is not None:
            loud_local.record_stream(self.side)
        return self.seq

    def latest(self, n: Optional[int] = None):
        """Newest complete vector of every rank, without waiting for anybody: ``(values [world, n], seqs [world])``
        (int32 sequence number per row; 0 and a NaN row for a rank that has not published yet).  The result lives on
        the side stream: call :meth:`wait` (or synchronise) before consuming it on another stream."""
        if n is None:
            n = self._n[self.seq] if self.seq in self._n else self.n_max
        out = torch.empty(self.world, n, dtype=torch.float32, device=self.device)
        seqs = torch.zeros(self.world, dtype=torch.int32, device=self.device)
        with self._on_side():
            self.launches += self.lib.call(self.lib.b2a_peer_latest_f32, self._ct.c_void_p(self.local), self.world, n,
                                           self.n_max, self._ct.c_void_p(out.data_ptr()),
                                           self._ct.c_void_p(seqs.data_ptr()), self._stream_ptr())
        return out, seqs

    def collect(self, seq: int, return_seqs: bool = False):
        """Lock-step gather ``[world * n]`` of sequence number ``seq`` (bounded device-side wait until every rank has
        published it; a rank that died or is more than three steps ahead yields a NaN row).  Side stream."""
        assert 1 <= seq <= self.seq, (seq, self.seq)
        n = self._n.get(seq, self.n_max)
        out = torch.empty(self.world * n, dtype=torch.float32, device=self.device)
        seqs = torch.zeros(self.world, dtype=torch.int32, device=self.device)
        with self._on_side():
            self.launches += self.lib.call(self.lib.b2a_peer_collect_f32, self._ct.c_void_p(self.local), self.world, n,
                                           self.n_max, seq, self._ct.c_void_p(out.data_ptr()),
                                           self._ct.c_void_p(seqs.data_ptr()), self._stream_ptr())
        return (out, seqs) if return_seqs else out

    def status(self) -> int:
        """Last sequence number a ``collect`` gave up on (0: none).  Synchronises the side stream."""
        st = torch.zeros(1, dtype=torch.int32, device=self.device)
        with self._on_side():
            self.lib.check(self.lib.b2a_peer_status(self._ct.c_void_p(self.local), self.world, self.n_max,
                                                    self._ct.c_void_p(st.data_ptr()), self._stream_ptr()))
        self.wait()
        return int(st.item())

    def wait(self):
        """Make the caller's current stream wait for everything issued on the exchange's side stream."""
        if self.side is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.side)

    def close(self):
        if getattr(self, "local", None) is None:
            return
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)  # nobody still stores into a buffer that is about to go away
        for p in self._opened:
            self.lib.b2a_peer_buffer_close(self._ct.c_void_p(p))
        self.lib.b2a_peer_buffer_destroy(self._ct.c_void_p(self.local))
        self.local = None
