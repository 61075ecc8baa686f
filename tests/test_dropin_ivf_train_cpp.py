"""IvfIndex's training upsert and RebuildCentroids through the IVF adapter's GpuIvfMap::TrainAndFill (reindexer_b200/host/gpu_ivf.h),
compiled against the reference's own vendored FAISS headers: the same lists in FAISS's direct map and on the device, no import before
the first search, recall within 0.02 of the CPU-trained index (tests/cpp/dropin_ivf_train_check.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_ivf_train_check")


def test_ivf_train_adapter_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "ivf_train.mk", "ivf_train"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_ivf_train_adapter_matches_reference_on_gpu():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_ivf_train_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") == 3
