"""torchrun script (world >= 2, one GPU per rank): the sharded range batch (rxgpu_sharded_search_range_batch over NCCL) must return, on
every rank, exactly what ONE index holding all rows returns through rxgpu_search_range_batch -- the same totals, labels in the same order
and the same distance bits -- on the tensor-core filter path (a batch) and on the exact-scan path (few queries).
tests/test_sharded_range_gpu.py has the same checks with the ranks as threads of one process."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import reindexer_b200 as rx  # noqa: E402
from reindexer_b200.sharded import ShardedBruteforceSearch  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    for case, (metric, dim, rows, nq, tc, max_out) in enumerate([(rx.IP, 96, 20000, 128, 1, 400), (rx.L2, 64, 15000, 5, 0, 300)]):
        rng = np.random.default_rng(200 + case)  # the same stream on every rank
        total = rows * world
        allv = rng.normal(0, 0.25, size=(total, dim)).astype(np.float32)
        queries = rng.normal(0, 0.25, size=(nq, dim)).astype(np.float32)
        labels = (rng.permutation(total).astype(np.uint64) << np.uint64(32)) + np.uint64(5)  # label order is not shard order
        full = rx.GpuBruteforceSearch(metric, dim, total, device=local)
        full.add_points(labels, allv)
        full.set_tensor_core_filter(2)
        d, _, _ = full.search_knn(queries, 100)
        radii = np.ascontiguousarray(d[np.arange(nq), np.array([1, 10, 100])[np.arange(nq) % 3] - 1])
        D0, L0, N0 = full.search_range_batch(queries, radii, max_out)
        shard = rx.GpuBruteforceSearch(metric, dim, rows, device=local)
        shard.add_points(labels[rank * rows:(rank + 1) * rows], allv[rank * rows:(rank + 1) * rows])
        shard.set_tensor_core_filter(tc)
        s = ShardedBruteforceSearch(shard, rows)
        assert s.comm is not None
        D1, L1, N1 = s.search_range_batch(queries, radii, max_out)
        st = rx.last_search_stats()
        assert st["tc_used"] == tc and st["tc_fallbacks"] == 0, (case, rank, st)
        D2, L2, N2 = s.search_range_batch(torch.from_numpy(queries).cuda(), radii, max_out)
        valid = np.arange(max_out)[None, :] < np.minimum(N0, max_out)[:, None]
        for D, L, N in ((D1, L1, N1), (D2, L2, N2)):
            assert (N == N0).all(), (case, rank)
            assert (~valid | (L == L0)).all(), (case, rank, np.argwhere(valid & (L != L0))[:4])
            assert (~valid | (D.view(np.uint32) == D0.view(np.uint32))).all(), (case, rank)
        assert N0.sum() >= 9 * nq, (case, N0.sum())
        s.comm.close()
        full.close()
        shard.close()
        dist.barrier()
    if rank == 0:
        print("mp_sharded_range_nccl ok", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
