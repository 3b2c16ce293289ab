"""TEST INFRASTRUCTURE — stand-in for the absent `sparse_dot_topn` wheel so the
UNMODIFIED reference (string_grouper/string_grouper.py:12) can be
imported by oracle/make_golden.py and the reference-suite pin test."""
import os
import sys

_root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _root not in sys.path:
    sys.path.insert(0, _root)
from oracle.sdt import sp_matmul_topn, zip_sp_matmul_topn  # noqa: E402,F401

__version__ = "0+oracle"
