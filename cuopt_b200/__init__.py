"""cuopt_b200 — H100-native (sm_90a) PDLP behind the libcuopt C ABI.

The product is `cuopt_b200/lib/libcuopt.so` (C ABI in include/); this package only holds the build recipe
(`build.py`) and the ctypes stub (`capi.py`) that tests and bench.py use to cross that boundary.
"""
from . import build  # noqa: F401
