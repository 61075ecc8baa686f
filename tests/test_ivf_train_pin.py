"""CPU check of the k-means plan of rxgpu_ivf_train (rxgpu_kmeans_plan, host only): the sample and the initial centroids come from the
same std::mt19937 draws as FAISS's Clustering::train -- subsample_training_set with rand_perm(n, seed) when n exceeds
nlist x max_points_per_centroid, then rand_perm(sample size, seed + 1) for the initial centroids, or the first nlist input rows when the
sample size equals nlist.  Compared with the reference FAISS's own rand_perm (tests/ivf_train_oracle.py)."""
import ivf_train_oracle as TO
import numpy as np
import pytest

import reindexer_b200 as rx

ERR_PARAMS = 3


def faiss_plan(n, nlist, seed, maxppc):
    if n > nlist * maxppc:
        sample = TO.rand_perm(n, seed)[:nlist * maxppc]
    else:
        sample = np.arange(n, dtype=np.int32)
    if len(sample) == nlist:  # Clustering.cpp's corner case: the first nlist rows of the input itself
        return sample, np.arange(nlist, dtype=np.int32)
    return sample, sample[TO.rand_perm(len(sample), seed + 1)[:nlist]]


@pytest.mark.skipif(not TO.available(), reason="needs tests/cpp/_build/libivf_train_oracle.so (reference FAISS build)")
@pytest.mark.parametrize("nlist", [1, 7, 100])
@pytest.mark.parametrize("seed", [0, 1234, 99991, 2**31 - 1])
def test_plan_equals_faiss_rand_perm(nlist, seed):
    for n in sorted({nlist, nlist + 1, 39 * nlist, 256 * nlist, 256 * nlist + 1, 10**6}):
        s, i = rx.kmeans_plan(n, nlist, seed)
        ws, wi = faiss_plan(n, nlist, seed, 256)
        assert (s == ws).all() and (i == wi).all(), (n, nlist, seed)


@pytest.mark.skipif(not TO.available(), reason="needs tests/cpp/_build/libivf_train_oracle.so (reference FAISS build)")
@pytest.mark.parametrize("maxppc", [1, 2, 39])
def test_plan_other_sample_caps(maxppc):
    nlist = 50
    for n in (nlist, 3 * nlist, maxppc * nlist, maxppc * nlist + 1, 1000 * nlist):
        s, i = rx.kmeans_plan(n, nlist, 17, maxppc)
        ws, wi = faiss_plan(n, nlist, 17, maxppc)
        assert (s == ws).all() and (i == wi).all(), (n, maxppc)
    # subsampled down to exactly nlist points: FAISS copies the first nlist INPUT rows, not the sample's
    s, i = rx.kmeans_plan(10 * nlist, nlist, 17, 1)
    assert len(s) == nlist and (i == np.arange(nlist)).all()


@pytest.mark.parametrize("args", [(10, 20, 1234, 256), (10, 0, 1234, 256), (10**6, 131073, 1234, 256), (100, 10, -1, 256), (100, 10, 5, 0)])
def test_plan_rejects_what_faiss_rejects(args):
    n, nlist, seed, maxppc = args
    with pytest.raises(rx.RxGpuError) as e:
        rx.kmeans_plan(n, nlist, seed, maxppc)
    assert e.value.code == ERR_PARAMS
