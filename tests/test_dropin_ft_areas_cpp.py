"""The highlight-area side of the ft_fast adapter (reindexer_b200/host/gpu_ft_merge.h: MergeAreas, MergeableAreas) compiled against
the reference's own headers and diffed against ft::Merger<IdCont, MergeDataAreas<Area>, OffsetT> (tests/cpp/dropin_ft_areas_check.cc)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "_build", "dropin_ft_areas_check")


def test_areas_adapter_compiles_against_reference_headers():
    if not os.path.isdir("/root/reference/cpp_src"):
        pytest.skip("reference tree not present on this box (the prebuilt binary is used by the gpu test)")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "ref", "port"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "areas.mk", "areas"])
    assert os.path.exists(BIN)


@pytest.mark.gpu
def test_areas_adapter_matches_reference_merger_on_gpu():
    if not os.path.exists(BIN):
        pytest.skip("tests/cpp/_build/dropin_ft_areas_check was not built (needs /root/reference at build time)")
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "MISMATCH" not in out.stdout and out.stdout.count("MATCH") >= 4
