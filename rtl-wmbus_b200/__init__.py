"""rtl-wmbus_b200 -- CUDA (H100, sm_90a) replacement for the per-sample DSP hot path of rtl-wmbus.

The product is the C-ABI shared library ``libwmbus_b200.so`` (include/wmbus_b200.h) built
from ``csrc/`` for sm_90a, plus the C host program ``rtl_wmbus_b200`` that keeps the
reference's stdin-cu8 -> stdout-datagram command line.  This Python package is only the
thin ctypes mirror of that ABI used by the tests and the benchmark; there is no Python or
CPU implementation of the path behind it -- loading fails loudly when the CUDA library is
missing.

Import with ``importlib.import_module("rtl-wmbus_b200")`` (the directory name carries the
reference's hyphen).
"""
from .capi import (WmbOpts, WmbStats, WmbFrame, WmbLineInfo, WmbDecoded, WmbRepaired, WmbRepairRecord, WmbusB200, load_library, library_path, build,
                   opts_from_flags, line_info_dtype, burst_dtype, BURST_CONTINUED, BURST_CUT, BURST_AT_END, spectrum_dtype,
                   line_quality_dtype, burst_quality_dtype, snippet_dtype, telegram_dtype, group_telegrams, LIB_NAME)

__all__ = ["WmbOpts", "WmbStats", "WmbFrame", "WmbLineInfo", "WmbDecoded", "WmbRepaired", "WmbRepairRecord", "WmbusB200", "load_library", "library_path", "build",
           "opts_from_flags", "line_info_dtype", "burst_dtype", "BURST_CONTINUED", "BURST_CUT", "BURST_AT_END", "spectrum_dtype",
           "line_quality_dtype", "burst_quality_dtype", "snippet_dtype", "telegram_dtype", "group_telegrams", "LIB_NAME"]
