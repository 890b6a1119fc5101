"""Two-process, two-GPU test of the NVLink peer-memory loudness exchange (audiotools_b200/parallel.py
PeerLoudnessExchange over csrc/peer.cu) against an NCCL all-gather of the same vectors.  Needs >= 2 GPUs:
skipped on a machine with one GPU (`python -m pytest tests/test_peer_exchange_gpu.py -m gpu` on two); the
same comparison is asserted, untimed, inside `bench.py` at every N > 1 so every multi-GPU bench run covers it."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import __graft_entry__ as graft

    graft.build()
    from audiotools_b200 import AudioSignal
    from audiotools_b200.parallel import PeerLoudnessExchange

    ok = True
    ex = PeerLoudnessExchange(n_max=64)
    g = torch.Generator().manual_seed(100 + rank)
    x = (0.1 * torch.randn(8, 2, 44100, generator=g)).cuda()
    # (a) lock-step: every step's vector, collected exactly, equals NCCL's all_gather of the same vector
    pending = None
    for step in range(9):
        loud = AudioSignal(x * (1 + 0.1 * step), 44100).loudness().contiguous()
        ref = torch.empty(world * loud.numel(), device=loud.device)
        dist.all_gather_into_tensor(ref, loud)
        if pending is not None:  # consume one step late
            seq_prev, ref_prev = pending
            got, seqs = ex.collect(seq_prev, return_seqs=True)
            ex.wait()
            ok &= torch.equal(got, ref_prev) and seqs.tolist() == [seq_prev] * world
        pending = (ex.put(loud), ref)
    got = ex.collect(pending[0])
    ex.wait()
    ok &= torch.equal(got, pending[1])
    # (b) no per-step collective, rank 1 deliberately delayed (ADVICE r1): `latest` never waits and only ever returns a
    #     vector that really is the one published under the sequence number it reports
    torch.cuda.synchronize()
    dist.barrier()
    base = ex.seq
    table = {}
    for step in range(12):
        if rank == 1 and step % 3 == 0:
            torch.cuda._sleep(20_000_000)  # ~10 ms of skew on the compute stream
        v = (torch.arange(16, device="cuda", dtype=torch.float32) + 1000.0 * rank + (base + step + 1)).contiguous()
        seq = ex.put(v)
        ok &= seq == base + step + 1
        vals, seqs = ex.latest(16)
        table[step] = (vals, seqs)
    ex.wait()
    torch.cuda.synchronize()
    for step, (vals, seqs) in table.items():
        for r in range(world):
            s_r = int(seqs[r])
            if s_r == 0:
                continue
            ok &= base < s_r <= base + 12 or s_r <= base
            if s_r > base:
                expect = torch.arange(16, device="cuda", dtype=torch.float32) + 1000.0 * r + s_r
                ok &= torch.equal(vals[r], expect)
        ok &= int(seqs[rank]) == base + step + 1  # a rank always sees its own newest vector
    dist.barrier()
    vals, seqs = ex.latest(16)
    ex.wait()
    ok &= seqs.tolist() == [base + 12] * world
    ok &= ex.status() == 0
    torch.cuda.synchronize()
    ex.close()
    dist.destroy_process_group()
    q.put((rank, bool(ok)))


@pytest.mark.gpu
def test_peer_exchange_matches_nccl_all_gather():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, 29533, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    res = dict(q.get(timeout=10) for _ in range(2))
    assert res == {0: True, 1: True}
