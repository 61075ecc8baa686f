"""The IVF adapter (reindexer_b200/host/gpu_ivf.h) over a faiss::IndexIVFFlat with 20 000 centroids, compiled against the reference's
own vendored FAISS headers and diffed against faiss::IndexIVFFlat through upserts and deletes (search at k = 10 and 1000, range_search;
tests/cpp/dropin_ivf_many_centroids_check.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_ivf_many_centroids_check")


def test_ivf_many_centroids_adapter_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "ivf_many_centroids.mk", "ivf_many_centroids"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_ivf_many_centroids_adapter_matches_reference_faiss_on_gpu():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_ivf_many_centroids_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") == 3
