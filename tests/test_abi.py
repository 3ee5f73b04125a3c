"""The C-ABI library builds for sm_90a without a GPU, loads, and exports every symbol include/hcp_b200.h declares."""
import ctypes
import os
import re

import hcp_diffusion_b200 as pkg
from hcp_diffusion_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_exports_header_symbols():
    path = pkg.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, "include", "hcp_b200.h")).read()
    declared = set(re.findall(r"\b(hcp_[a-z0-9_]+)\s*\(", header))
    declared -= {"hcp_status"}
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for sym in declared:
        assert hasattr(lib, sym), sym
    lib.hcp_version.restype = ctypes.c_int
    assert lib.hcp_version() >= 1
    lib.hcp_last_error_string.restype = ctypes.c_char_p
    assert lib.hcp_last_error_string() is not None


def test_struct_sizes_match_the_header():
    # the ctypes mirrors must have the C layout: spot-check through sizes computed by hand from the header
    assert ctypes.sizeof(_lib.GemmArgs) == 8 + 3 * 8 * 6 + 2 * 8 + 4 * 8 + 2 * 8 + 2 * 8 + 8 + 16 + 3 * 8
    assert ctypes.sizeof(_lib.LoraJob) == 8 * 2 + 4 * 7 + 4 + 8 * 4
    assert ctypes.sizeof(_lib.ConvArgs) == 2 * 8 + 5 * 8 + 8 + 5 * 8 + 16 + 4 * 8 + 8        # + w_tiled (int32, padded)
    assert ctypes.sizeof(_lib.LoraMergeJob) == 8 + 4 * 8 * 2 + 4 * 4 * 2 + 6 * 4 + 2 * 4 + 2 * 8
    assert ctypes.sizeof(_lib.LoraConvJob) == 8 + 6 * 4 + 2 * 8
