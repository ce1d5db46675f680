#!/usr/bin/env python
"""Record tests/golden/ref_digests.npz and tests/golden/ref_digests_repeats.npz (test_repeats_cpu.py's checks): runs the
differential tests with BARB200_RECORD_REF=1, so that every check calls the unmodified reference (oracle/_ref, built by
oracle/Makefile where the reference sources exist), compares it with the checked implementation directly and stores the digest of the reference's answer (tests/_refgold.py).

  python scripts/make_golden_ref_digests.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["BARB200_RECORD_REF"] = "1"
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pytest  # noqa: E402

import _reflib as R  # noqa: E402


def main():
    assert R.have_ref() and R.have_bar_ref() and R.have_pecan_ref(), "build oracle/_ref first (make -C oracle)"
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_oracle_vs_ref.py"),
                      os.path.join(ROOT, "tests", "test_poa_params_cpu.py"),
                      os.path.join(ROOT, "tests", "test_repeats_cpu.py") + "::test_oracle_equals_reference",
                      os.path.join(ROOT, "tests", "test_repeats_cpu.py") + "::test_key_capacity_cases_equal_reference",
                      os.path.join(ROOT, "tests", "test_repeats_cpu.py") + "::test_long_window_equals_reference",
                      os.path.join(ROOT, "tests", "test_repeats_cpu.py") + "::test_windows_and_two_ends_equal_reference",
                      os.path.join(ROOT, "tests", "test_pecan_cpu.py") + "::test_oracle_vs_reference_random"])
    if rc != 0:
        return int(rc)
    import _refgold
    import test_repeats_cpu
    print("%d digests -> %s" % (_refgold.save(), _refgold.PATH))
    print("%d digests -> %s" % (test_repeats_cpu.save_digests(), test_repeats_cpu.DIGESTS))
    return 0


if __name__ == "__main__":
    sys.exit(main())
