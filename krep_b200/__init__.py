"""krep_b200 — H100-native scan engine behind krep's search_func_t boundary.

The product is the C-ABI shared library built from krep_b200/csrc (see include/krep_b200.h);
this package only holds the build recipe and the ctypes plumbing used by tests and bench.py.
"""
from . import abi  # noqa: F401

__version__ = "0.1.0"
