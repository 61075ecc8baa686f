"""CPU check of the IVF oracle over given centroids and lists (tests/ivf_lists_oracle.py): on integer-valued L2 data every distance is
exact, so FAISS' answer must equal a numpy model that probes the nprobe nearest lists under (distance, centroid id) and keeps the k
nearest of their rows; adds go to the list FAISS' quantizer picks, removes leave the lists."""
import ivf_lists_oracle as LO
import numpy as np
import pytest

pytestmark = pytest.mark.skipif(not LO.available(), reason="needs tests/cpp/_build/libivf_lists_oracle.so (reference FAISS build)")


def int_rows(seed, n, dim):
    return np.random.default_rng(seed).integers(-4, 4, size=(n, dim)).astype(np.float32)


def l2(x, q):
    return ((x.astype(np.float64) - q.astype(np.float64)) ** 2).sum(1)


def test_given_lists_match_numpy_model():
    dim, nlist, n = 8, 20000, 40000
    rng = np.random.default_rng(1)
    cents, vecs = int_rows(5, nlist, dim), int_rows(6, n, dim)
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(3)
    list_nos = rng.integers(0, nlist, n).astype(np.int64)
    ref = LO.ListsIvf(0, cents, list_nos, labels, vecs)
    assert (ref.list_of(labels[:500]) == list_nos[:500]).all()
    for q in int_rows(7, 4, dim):
        cd = l2(cents, q)
        for nprobe in (7, 300):
            probed = np.lexsort((np.arange(nlist), cd))[:nprobe]
            rows = np.nonzero(np.isin(list_nos, probed))[0]
            want = np.sort(l2(vecs[rows], q))[:50]
            d, l = ref.search(q, 50, nprobe)
            assert len(d) == len(want) and (d == want.astype(np.float32)).all(), nprobe
            assert set(l.tolist()) <= set(labels[rows].tolist())
    new = int_rows(8, 10, dim)
    new_labels = np.arange(10, dtype=np.uint64) | np.uint64(1 << 62)
    ref.add(new_labels, new)
    got = ref.list_of(new_labels)
    for v, c in zip(new, got):
        dv = l2(cents, v)
        assert c == np.lexsort((np.arange(nlist), dv))[0]  # the quantizer's nearest centroid
    ref.remove(int(new_labels[0]))
    with pytest.raises(AssertionError):
        ref.list_of(new_labels[:1])
