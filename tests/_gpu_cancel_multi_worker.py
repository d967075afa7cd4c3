"""One rank of the multi-GPU cancel test: push a skewed shard, cancel a first list on rank 0, b9_rebalance (NCCL), cancel a
second list on every rank, drain, dump."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    rank, world, out_dir = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    from beta9_b200.device_queue import DeviceQueue
    from tests._rebalance_worker import shard_for
    q = DeviceQueue(device=rank, ring_bytes=1 << 28, ring_tasks=1 << 18, max_drain_tasks=1 << 18, max_result_bytes=1 << 28)
    idf = os.path.join(out_dir, "nccl_id.bin")
    if rank == 0:
        uid = DeviceQueue.comm_unique_id()
        with open(idf + ".tmp", "wb") as f:
            f.write(uid)
        os.replace(idf + ".tmp", idf)
    else:
        t0 = time.time()
        while not os.path.exists(idf):
            if time.time() - t0 > 120:
                raise SystemExit("no NCCL id")
            time.sleep(0.05)
        uid = open(idf, "rb").read()
    q.comm_init(uid, rank, world)
    shards = [shard_for(r, world, "rank0_heavy") for r in range(world)]
    b = shards[rank]
    q.push_batch(b.task_ids, b.payload, b.offsets)
    # the first list: every 5th task of rank 0's shard, cancelled where it was pushed, before the exchange
    first = shards[0].task_ids[::5]
    if rank == 0:
        m1, o1 = q.cancel(first)
        assert m1 == first.shape[0] and np.all(o1 == 1), (m1, o1)
    q.rebalance()
    # the second list, given to every rank: every 7th task of every shard (some of them in the first list too)
    second = np.concatenate([s.task_ids[1::7] for s in shards])
    m2, o2 = q.cancel(second)
    r = q.drain("identity")
    np.savez(os.path.join(out_dir, f"cancel_rank{rank}.npz"), ids=r.task_ids, status=r.status, has=r.has_result, lens=r.lengths,
             payload=r.fifo_payload(), before_ids=b.task_ids, before_offsets=b.offsets, before_payload=b.payload,
             first=first, second=second, marked2=np.int64(m2), outcome2=o2)
    q.close()


if __name__ == "__main__":
    main()
