"""The drop-in adapters (reindexer_b200/host/gpu_bruteforce.h, gpu_hnsw.h, gpu_ivf.h) searched by six reader threads under a shared lock,
with a writer taking it exclusive between rounds, compiled against the reference's own headers (tests/cpp/dropin_concurrency_check.cc):
every reader's answer must equal the adapter's serial answer at the same epoch, and that answer the reference map's."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_concurrency_check")


def test_concurrency_check_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "concurrency.mk", "concurrency"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_adapters_under_a_shared_lock_match_serial_answers_and_the_reference():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_concurrency_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") == 6, out.stdout
