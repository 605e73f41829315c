"""Worker of tests/test_gpu_nccl_fallback.py — one process per GPU under torchrun (NCCL).  NOT a pytest module.

Every rank owns a contiguous ring-0 range of the virtual nodes, as in tests/nccl_worker.py.  One scenario:

  fallback  A split vote with no fast quorum: a fixed set of nodes crashes in every receiver's eyes, and half of the receivers
            (even global ring-0 position) never hear about one more crashed subject `x`, so two proposals get about n/2 votes
            each and the sharded fast-round tally does not decide.  Every rank registers its receivers' votes into its
            PaxosAcceptors shard (acceptor_begin = receiver_begin) and runs the classic round through the sharded tallies
            (Paxos.handlePhase1bFromAcceptorShards / handlePhase2bFromAcceptorShards over the NCCL communicator).  Every rank
            must get the same cval, trigger index and decision, equal to those of a single-handle round that rank 0 runs on
            one PaxosAcceptors over all n acceptors, built from the gathered per-receiver outputs.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

K, H, L = 10, 9, 4


def main():
    import torch
    import torch.distributed as dist
    import rapid_b200 as rb
    from rapid_b200 import workloads as W

    n = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports, device=local)
    hi, lo = W.node_ids(0, n)
    cfg = view.getCurrentConfigurationId(hi, lo)
    ring0 = view.getRing(0)
    obs, _ = view.tables()
    begin = rank * n // world
    R = (rank + 1) * n // world - begin
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid.copy_(torch.from_numpy(rb.NcclComm.unique_id()))
    dist.broadcast(uid, 0)
    comm = rb.NcclComm(rank, world, uid.cpu().numpy(), local)

    base = W.pick_smallest(n, 12, W.SEED + 77)                   # crashed in every receiver's eyes
    x = next(i for i in range(n) if i not in set(base.tolist()))
    failed = np.append(base, x).astype(np.int32)
    cells = W.crash_cells(obs, np.sort(failed), n)
    src, dst, ring, status = cells["src"], cells["dst"], cells["ring"], cells["status"]
    bl = np.zeros(n, np.uint8)
    bl[failed] = 1
    blocked = W.blocked_by_receiver(bl, ring0, begin, R)
    deaf = (begin + np.arange(R)) % 2 == 0
    words = (R + 31) // 32
    row_deaf = np.zeros(words, np.uint32)
    hear = np.nonzero(~deaf)[0]
    np.bitwise_or.at(row_deaf, hear >> 5, (np.uint32(1) << (hear & 31).astype(np.uint32)))
    bitmap = np.where((dst == x)[:, None], row_deaf[None, :], np.full(words, 0xFFFFFFFF, np.uint32)[None, :]).astype(np.uint32)

    cl = rb.VirtualCluster(view, H, L, n_receivers=R, receiver_begin=begin)
    res = cl.handleBatch(cfg, src, dst, ring, status, blocked=blocked, bitmap=bitmap)
    t = rb.FastPaxos(cfg, n, sender_capacity=n, device=local).tallyCluster(cl, comm)
    assert not t.decided, "the split vote reached the fast quorum"

    # the classic round, sharded: this rank's acceptors are its receivers
    acc = rb.PaxosAcceptors(cfg, R, acceptor_begin=begin, device=local)
    acc.registerFastRoundVotesFrom(cl)
    px = rb.Paxos(cfg, n, device=local)
    assert px.startPhase1a(2, 7)
    acc.handlePhase1aMessage((2, 7))
    got = px.handlePhase1bFromAcceptorShards([acc], comm=comm, perm_seed=4321)
    assert got.proposed and got.n_messages == n
    acc.handlePhase2aMessage((2, 7), got.cval)
    dec = rb.Paxos(cfg, n, device=local).handlePhase2bFromAcceptorShards([acc], comm=comm, perm_seed=99)
    assert dec.decided
    mine = (got.trigger_index, got.cval, dec.decided_index, dec.decision)

    outs = [None] * world
    dist.all_gather_object(outs, (np.asarray(res.announced), np.asarray(res.proposal_hash), np.asarray(res.proposal_hash2),
                                  np.asarray(res.proposal_len), mine))
    assert all(o[4] == mine for o in outs), "ranks disagree: %r" % ([o[4] for o in outs],)
    if rank == 0:
        # the same round on one handle over all n acceptors, from the gathered per-receiver outputs (ranks in ring-0 order)
        ids = np.nonzero(np.concatenate([o[0] for o in outs]) != 0)[0].astype(np.int64)
        h1, h2, ln = (np.concatenate([o[k] for o in outs])[ids] for k in (1, 2, 3))
        assert len(set(h1.tolist())) == 2, "expected two proposals"
        one = rb.PaxosAcceptors(cfg, n, device=local)
        one.registerFastRoundVotes(ids, h1, ln, h2)
        rpx = rb.Paxos(cfg, n, device=local)
        rpx.startPhase1a(2, 7)
        assert one.handlePhase1aMessage((2, 7)) == n
        r1 = rpx.handlePhase1bFromAcceptors(one, perm_seed=4321)
        assert one.handlePhase2aMessage((2, 7), r1.cval) == n
        r2 = rb.Paxos(cfg, n, device=local).handlePhase2bFromAcceptors(one, perm_seed=99)
        assert (r1.trigger_index, r1.cval, r2.decided_index, r2.decision) == mine, (r1, r2, mine)
        print("nccl fallback worker ok: world=%d n=%d fast round undecided (%d votes received); classic round triggered at %d, "
              "decided at %d" % (world, n, t.votes_received, got.trigger_index, dec.decided_index), flush=True)
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
