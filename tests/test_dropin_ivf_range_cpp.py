"""The IVF adapter (reindexer_b200/host/gpu_ivf.h) answering range_search for a batch of queries, compiled against the reference's own
vendored FAISS headers and diffed against faiss::IndexIVFFlat and against one-query adapter calls through upserts and deletes
(tests/cpp/dropin_ivf_range_check.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_ivf_range_check")


def test_ivf_range_adapter_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "ivf_range.mk", "ivf_range"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_ivf_range_adapter_matches_reference_faiss_on_gpu():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_ivf_range_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") == 3
