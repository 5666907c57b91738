"""Regenerate tests/golden/ref_v1.npz: the outputs of THE REFERENCE'S OWN SOURCES for every input the tests give them.

The tests compare the oracle and the kernels with the reference's factor / preintegration / marginalization / FeatureManager
sources through oracle_lib.RefBackend, which replays this file, so that the comparison runs wherever the suite runs.  This
script runs those tests once with the compiled sources (oracle/_ref/libcerberus_ref.so) and stores every call:

  make -C oracle ref REF=<Cerberus checkout>/src
  python tests/golden/make_ref_golden.py

The GPU-tier tests among them run on the CPU kernel simulator here: their reference inputs do not depend on the device.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import pytest                                       # noqa: E402
from cerberus_b200 import lib                       # noqa: E402
import oracle_lib                                   # noqa: E402
from helpers import SIM_LIB, sim_backend            # noqa: E402

TESTS = ["tests/test_reference_pin.py", "tests/test_parity_r2.py"]


class _SimulatedDevice(lib.Backend):
    def __init__(self, cfg=None, lib_path=None):
        super().__init__(cfg, lib_path or SIM_LIB)


def main():
    if oracle_lib.ref_lib() is None:
        sys.exit("oracle/_ref/libcerberus_ref.so is not built: make -C oracle ref REF=<Cerberus checkout>/src")
    sim_backend().close()                           # builds the simulator if needed
    oracle_lib.RefBackend.record = True
    lib.Backend = _SimulatedDevice
    rc = pytest.main(["-p", "no:xdist", "-p", "no:cacheprovider", "-q", "-m", "", "-k", "not stress", "--rootdir", ROOT] + [os.path.join(ROOT, t) for t in TESTS])
    if rc != 0:
        sys.exit(f"the tests failed with the live reference sources (pytest exit code {rc}); nothing written")
    oracle_lib.GOLDEN.save()
    n = sum(len(v) for v in oracle_lib.GOLDEN.load().values())
    print(f"wrote {oracle_lib.GOLDEN_REF}: {n} calls, {os.path.getsize(oracle_lib.GOLDEN_REF)} bytes")


if __name__ == "__main__":
    main()
