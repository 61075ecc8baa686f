"""Multi-GPU brute-force KNN: the namespace is sharded by internal-row range, one process per GPU (torch.distributed),
each rank scans its own shard with the fused distance + top-k kernel, and the per-shard top-(k+1) lists are exchanged with ONE
all-gather (NCCL over NVLink/NVSwitch on GPUs; gloo in the CPU tests) and merged under the reference's comparator.

SURVEY.md §8e: shard g holds global internal rows [base[g], base[g+1]) so that the reference's order-dependent tie rule
(bruteforce.cc:103-127) can still be replayed globally: a tie straddling the k-th place triggers one extra "tie rows" scan on
every shard and a second all-gather.  The exchange is Q*(k+1)*16 B per rank -- latency-bound, not bandwidth-bound.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from . import binding as B


class ShardedBruteforceSearch:
    """Collective object: every rank constructs it with its local shard and calls the same methods in the same order."""

    def __init__(self, local_index, shard_rows: int, group=None, device=None, local_search=None, local_tie_rows=None):
        self.idx = local_index
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.device = device if device is not None else (torch.device("cuda", torch.cuda.current_device())
                                                         if torch.cuda.is_available() else torch.device("cpu"))
        # global internal-row base of every shard (rows are appended shard by shard)
        sizes = self._all_gather_small(torch.tensor([shard_rows], dtype=torch.int64)).numpy().ravel()
        self.shard_base = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64)
        self.total_rows = int(sizes.sum())
        self._local_search = local_search or self._device_search
        self._local_tie_rows = local_tie_rows or self._device_tie_rows
        self.replay_ties = True  # the brute-force map reproduces the reference's heap tie rule; approximate maps have none
        # On GPUs the whole search is ONE C-ABI call per rank (rxgpu_sharded_search_knn: local scan, ncclAllGather, device merge, tie
        # replay from the filter's candidate lists); torch.distributed only ships the NCCL unique id once.  The Python exchange below
        # remains for the CPU (gloo) tests of the merge / tie logic and for maps without a C-side sharded call (HNSW shards).
        self.comm = None
        if local_search is None and local_tie_rows is None and type(self) is ShardedBruteforceSearch and self.device.type == "cuda":
            dev = self.device.index if self.device.index is not None else torch.cuda.current_device()
            if self.world > 1:
                ident = torch.zeros(B.COMM_ID_BYTES, dtype=torch.uint8)
                if self.rank == 0:
                    ident = torch.frombuffer(bytearray(B.comm_unique_id()), dtype=torch.uint8).clone()
                ident = ident.to(self.device)
                dist.broadcast(ident, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0, group=self.group)
                self.comm = B.ShardComm(self.world, self.rank, bytes(ident.cpu().numpy().tobytes()), dev)
            else:
                self.comm = B.ShardComm(1, 0, None, dev)

    # -- plumbing ----------------------------------------------------------------------------------------------------------
    def _all_gather_small(self, t: torch.Tensor) -> torch.Tensor:
        if self.world == 1:
            return t.reshape(1, *t.shape).cpu()
        t = t.to(self.device).contiguous()
        out = torch.empty((self.world * t.numel(),), dtype=t.dtype, device=self.device)
        dist.all_gather_into_tensor(out, t.reshape(-1), group=self.group)
        return out.view(self.world, *t.shape).cpu()

    def _device_search(self, d_queries: torch.Tensor, k1: int):
        nq = d_queries.shape[0]
        od = torch.zeros((nq, k1), dtype=torch.float32, device=self.device)
        oi = torch.zeros((nq, k1), dtype=torch.int32, device=self.device)
        ol = torch.zeros((nq, k1), dtype=torch.int64, device=self.device)
        oc = torch.zeros((nq,), dtype=torch.int32, device=self.device)
        self.idx.search_knn_device(nq, d_queries.data_ptr(), k1, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream)
        return od, oi, ol, oc

    def _device_tie_rows(self, d_query: torch.Tensor, dstar: float, k: int):
        od = torch.zeros((k,), dtype=torch.float32, device=self.device)
        oi = torch.zeros((k,), dtype=torch.int32, device=self.device)
        ol = torch.zeros((k,), dtype=torch.int64, device=self.device)
        oc = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self.idx.search_tie_rows_device(d_query.data_ptr(), dstar, k, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream)
        return od, oi, ol, oc

    # -- search ------------------------------------------------------------------------------------------------------------
    def search_knn(self, queries, k: int):
        """queries: host ndarray [nq, dim] or device tensor (identical on every rank).  Returns (dist, label, count) on every
        rank, best-first, reference tie rule applied globally."""
        if self.comm is not None:  # the product path: one C-ABI call per rank
            if isinstance(queries, np.ndarray):
                return self.comm.search_knn(self.idx, queries, k)
            assert queries.is_cuda and queries.dtype == torch.float32 and queries.is_contiguous()
            torch.cuda.current_stream().synchronize()  # the library runs on its own stream: the queries must be complete
            return self.comm.search_knn(self.idx, queries.data_ptr(), k, nq=queries.shape[0])
        if isinstance(queries, np.ndarray):
            d_queries = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).to(self.device, non_blocking=True)
        else:
            d_queries = queries
        nq = d_queries.shape[0]
        k_eff = min(k, self.total_rows)
        if k_eff == 0 or nq == 0:
            return np.zeros((nq, k), np.float32), np.zeros((nq, k), np.uint64), np.zeros(nq, np.uint32)
        k1 = k_eff + 1
        od, oi, ol, oc = self._local_search(d_queries, k1)
        # ONE exchange: pack (dist, idx, label, count) into a single int64 tensor per rank
        packed = torch.empty((nq, 2 * k1 + 1), dtype=torch.int64, device=od.device)
        packed[:, :k1] = (od.view(torch.int32).to(torch.int64) & 0xFFFFFFFF) | (oi.to(torch.int64) << 32)
        packed[:, k1:2 * k1] = ol
        packed[:, 2 * k1] = oc.to(torch.int64)
        allp = self._all_gather_small(packed).numpy()  # [world, nq, 2*k1+1]
        lo = allp[:, :, :k1]
        D = (lo & 0xFFFFFFFF).astype(np.uint32).view(np.float32)
        I = ((lo >> 32) & 0xFFFFFFFF).astype(np.uint32)
        L = allp[:, :, k1:2 * k1].view(np.uint64)
        Cn = allp[:, :, 2 * k1].astype(np.uint32)
        rd, rg, rl, rc, need_tie = B.merge_shards(k_eff, D, I, L, Cn, self.shard_base)
        out_d = np.zeros((nq, k), np.float32)
        out_l = np.zeros((nq, k), np.uint64)
        out_d[:, :k_eff], out_l[:, :k_eff] = rd, rl
        for q in (np.nonzero(need_tie)[0] if self.replay_ties else ()):  # rare: bit-equal distances straddle the k-th place -> replay the reference's heap rule
            c = int(rc[q])
            dstar = float(rd[q, c - 1])
            td, ti, tl, tc = self._local_tie_rows(d_queries[q], dstar, k_eff)
            tp = torch.empty((2 * k_eff + 1,), dtype=torch.int64, device=td.device)
            tp[:k_eff] = (td.view(torch.int32).to(torch.int64) & 0xFFFFFFFF) | (ti.to(torch.int64) << 32)
            tp[k_eff:2 * k_eff] = tl
            tp[2 * k_eff] = tc.to(torch.int64)[0]
            allt = self._all_gather_small(tp).numpy()
            fd, fg, fl = [], [], []
            for s in range(self.world):
                n_s = int(allt[s, 2 * k_eff])
                lo_s = allt[s, :n_s]
                fd.append((lo_s & 0xFFFFFFFF).astype(np.uint32).view(np.float32))
                fg.append(((lo_s >> 32) & 0xFFFFFFFF).astype(np.uint64) + self.shard_base[s])
                fl.append(allt[s, k_eff:k_eff + n_s].view(np.uint64))
            fd, fg, fl = np.concatenate(fd), np.concatenate(fg), np.concatenate(fl)
            order = np.argsort(fg, kind="stable")[:k_eff]
            lower = rd[q, :c] < dstar
            td2, tl2 = B.tie_replay(k_eff, dstar, (rd[q, :c][lower], rg[q, :c][lower], rl[q, :c][lower]),
                                    (fd[order], fg[order], fl[order]))
            out_d[q, :len(td2)], out_l[q, :len(td2)] = td2, tl2
        return out_d, out_l, rc

    def search_range_batch(self, queries, radius, max_out: int):
        """queries: host ndarray [nq, dim] or device tensor (identical on every rank); radius: a scalar or [nq], map space.  Returns
        (dist [nq, max_out], label [nq, max_out], count [nq]) on every rank, as GpuBruteforceSearch.search_range_batch returns them for
        one index holding all rows.  One C-ABI call per rank (rxgpu_sharded_search_range_batch); there is no CPU exchange for it."""
        if self.comm is None:
            raise NotImplementedError("sharded range search runs on the GPUs only (rxgpu_sharded_search_range_batch)")
        if isinstance(queries, np.ndarray):
            return self.comm.search_range_batch(self.idx, queries, radius, max_out)
        assert queries.is_cuda and queries.dtype == torch.float32 and queries.is_contiguous()
        torch.cuda.current_stream().synchronize()  # the library runs on its own stream: the queries must be complete
        return self.comm.search_range_batch(self.idx, queries.data_ptr(), radius, max_out, nq=queries.shape[0])


class ShardedHnswSearch(ShardedBruteforceSearch):
    """Multi-GPU HNSW (SURVEY.md §8e): every GPU holds an independent sub-graph over its row range (built by the reference's
    inserter over that shard, imported with hnsw_import), all shards are searched for every query, and the per-shard top-k lists
    are merged exactly like the brute-force shards (one all-gather).  Recall is that of the per-shard graphs; there is no
    reference tie rule to replay (HierarchicalNSW::SearchKnn orders bit-equal distances by heap mechanics), results are ordered
    by (distance, global row)."""

    def __init__(self, local_index, shard_rows: int, ef: int, group=None, device=None, local_search=None):
        super().__init__(local_index, shard_rows, group=group, device=device, local_search=local_search)
        self.ef = ef
        self.replay_ties = False

    def _device_search(self, d_queries: torch.Tensor, k1: int):
        nq = d_queries.shape[0]
        od = torch.zeros((nq, k1), dtype=torch.float32, device=self.device)
        oi = torch.zeros((nq, k1), dtype=torch.int32, device=self.device)
        ol = torch.zeros((nq, k1), dtype=torch.int64, device=self.device)
        oc = torch.zeros((nq,), dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream().cuda_stream
        self.idx.hnsw_search_knn_device(nq, d_queries.data_ptr(), k1, max(self.ef, k1), od.data_ptr(), oi.data_ptr(), oc.data_ptr(),
                                        0, stream)
        self.idx.gather_labels_device(nq * k1, oi.data_ptr(), ol.data_ptr(), stream)
        return od, oi, ol, oc
