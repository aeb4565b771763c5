"""CPU check of the branch-free match codes (zippy_b200/csrc/zb_common.h) that k_lz's batch pass turns every match
into a packer record with: for every length 3..258 and every distance 1..32768 they give the same code and extra
value as zb_len_code / zb_len_base and zb_dist_code / zb_dist_base.  Built with g++ from
tests/native/lz_codes_units.cpp."""
import ctypes
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "lz_codes_units.cpp")


def test_branch_free_codes():
    tmp = tempfile.mkdtemp(prefix="lz_codes_units_")
    try:
        so = os.path.join(tmp, "liblz_codes_units.so")
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, SRC])
        assert ctypes.CDLL(so).t_codes_compare() == 0
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
