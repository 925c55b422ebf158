"""Programmatic dependent launch is how the specialised step is launched, not an option: no environment variable switches
it (tests/test_step_overlap_gpu.py checks on the GPU that the overlap of consecutive steps changes no result)."""
import os

import tds_b200

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tiny-differentiable-simulator_b200", "csrc")


def test_no_switch_for_programmatic_dependent_launch():
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh", ".h", ".cpp")):
            with open(os.path.join(CSRC, f)) as fh:
                assert "TDS_B200_PDL" not in fh.read(), f
    path = tds_b200.lib_path()
    if os.path.exists(path):
        with open(path, "rb") as fh:
            assert b"TDS_B200_PDL" not in fh.read()
