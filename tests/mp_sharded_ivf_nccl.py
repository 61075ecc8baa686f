"""torchrun script (world >= 2, one GPU per rank): one sharded IVF training (rxgpu_sharded_ivf_train over NCCL), each rank's list
assignment, one sharded KNN and one sharded range batch must give, on every rank, exactly what ONE index over all rows gives -- the same
centroid bits and per-iteration obj / nsplit, the same labels in the same order and the same distance bits.
tests/test_sharded_ivf_gpu.py has the same checks with the ranks as threads of one process."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import reindexer_b200 as rx  # noqa: E402
from reindexer_b200 import binding as B  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ident = torch.zeros(B.COMM_ID_BYTES, dtype=torch.uint8)
    if rank == 0:
        ident = torch.frombuffer(bytearray(B.comm_unique_id()), dtype=torch.uint8).clone()
    ident = ident.cuda()
    dist.broadcast(ident, src=0)
    comm = B.ShardComm(world, rank, bytes(ident.cpu().numpy().tobytes()), local)
    rng = np.random.default_rng(300)  # the same stream on every rank
    metric, dim, nlist, rows = rx.COS, 48, 64, 6000
    total = rows * world
    allv = rng.normal(0, 1, size=(total, dim)).astype(np.float32)
    labels = (rng.permutation(total).astype(np.uint64) << np.uint64(16)) + np.uint64(9)
    queries = rng.normal(0, 1, size=(50, dim)).astype(np.float32)
    cut = [total * r // world + (r * 37) % 500 for r in range(world)] + [total]  # uneven shards
    cut[0] = 0
    full = rx.GpuBruteforceSearch(metric, dim, 1, device=local)
    c0, s0 = full.ivf_train(nlist, allv, niter=5, max_points_per_centroid=80)
    full.ivf_add_assign(labels, allv)
    shard = rx.GpuBruteforceSearch(metric, dim, 1, device=local)
    a, b = cut[rank], cut[rank + 1]
    c1, s1 = comm.ivf_train(shard, nlist, allv[a:b], niter=5, max_points_per_centroid=80)
    assert (c1.view(np.uint32) == c0.view(np.uint32)).all(), rank
    assert [(t["obj"], t["nsplit"]) for t in s1] == [(t["obj"], t["nsplit"]) for t in s0], rank
    shard.ivf_add_assign(labels[a:b], allv[a:b])
    for k, nprobe in ((10, 8), (1000, 64)):
        D0, L0, C0 = full.ivf_search_knn_large_k(queries, k, nprobe)
        D1, L1, C1 = comm.ivf_search_knn(shard, queries, k, nprobe)
        assert (C1 == C0).all() and (L1 == L0).all() and (D1.view(np.uint32) == D0.view(np.uint32)).all(), (rank, k)
    d, _, _ = full.ivf_search_knn_large_k(queries, 100, nprobe=8)
    radii = np.ascontiguousarray(d[:, 60])
    D0, L0, N0 = full.ivf_search_range_batch(queries, radii, 8, 80)
    D1, L1, N1 = comm.ivf_search_range_batch(shard, queries, radii, 8, 80)
    valid = np.arange(80)[None, :] < np.minimum(N0, 80)[:, None]
    assert (N1 == N0).all() and (~valid | (L1 == L0)).all() and (~valid | (D1.view(np.uint32) == D0.view(np.uint32))).all(), rank
    comm.close()
    full.close()
    shard.close()
    dist.barrier()
    if rank == 0:
        print("mp_sharded_ivf_nccl ok", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
