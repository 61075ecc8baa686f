"""reindexer_b200 -- H100-native (sm_90a) replacement for Reindexer's float_vector KNN / ft_fast BM25 hot path.

The product is the C-ABI library ``librxgpu.so`` (include/rxgpu.h) and the C++ adapter under ``host/``; this package is
the thin Python driver used by tests, the benchmark and the multi-GPU (one process per GPU, torch.distributed) plumbing.
"""
from .binding import (COS, FLAG_HOST_MIRROR, IP, L2, GpuBruteforceSearch, GpuFtIndex, RxGpuError, ShardComm, device_count, hnsw_build_plan,
                      kmeans_plan, last_search_stats, lib, merge_shards, tie_replay)

__all__ = ["L2", "IP", "COS", "FLAG_HOST_MIRROR", "GpuBruteforceSearch", "GpuFtIndex", "RxGpuError", "ShardComm", "device_count", "hnsw_build_plan", "kmeans_plan", "last_search_stats", "lib",
           "merge_shards", "tie_replay"]
