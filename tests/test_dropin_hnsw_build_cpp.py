"""GpuHnsw<OnInsertions> with device building switched on (reindexer_b200/host/gpu_hnsw.h), compiled against the reference's own
headers: concurrent inserts from 8 threads in three rounds, host graph equal to the device graph, no import, recall within 0.01 of
HierarchicalNSW<OnInsertions>, an index-cache round trip, the reference's path for existing labels and tombstones, and the switch off
(tests/cpp/dropin_hnsw_build_check.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_hnsw_build_check")


def test_hnsw_build_adapter_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "hnsw_build.mk", "hnsw_build"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_hnsw_build_adapter_matches_reference_on_gpu():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_hnsw_build_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") == 12, out.stdout
