"""ctypes mirror of include/wmbus_b200.h (one wrapper class, no logic of its own)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libwmbus_b200.so"


class WmbOpts(C.Structure):
    _fields_ = [("decimation", C.c_uint32), ("accurate_atan", C.c_uint8), ("remove_dc", C.c_uint8),
                ("rla_enabled", C.c_uint8), ("t2_enabled", C.c_uint8), ("t1c1_enabled", C.c_uint8),
                ("s1_enabled", C.c_uint8), ("simultaneous", C.c_uint8), ("show_algorithm", C.c_uint8),
                ("chunk_samples", C.c_uint32), ("warmup_samples", C.c_uint32),
                ("max_batch_mib", C.c_uint32), ("manual_frames", C.c_uint32), ("reserved", C.c_uint32 * 2),
                ("carrier_25khz", C.c_int32 * 2), ("prefilter", C.c_uint32)]


class WmbFrame(C.Structure):
    _fields_ = [("sync_sample", C.c_uint64), ("ordinal", C.c_uint64), ("chain", C.c_uint8),
                ("algo", C.c_uint8), ("truncated", C.c_uint8), ("reserved", C.c_uint8),
                ("nbits", C.c_uint32), ("bits", C.POINTER(C.c_uint32))]


class WmbDecoded(C.Structure):
    """wmb_decoded (include/wmbus_b200_framer.h): one candidate's decode"""
    _fields_ = [("status", C.c_int), ("consumed", C.c_uint32), ("end_sample", C.c_uint64), ("mode", C.c_char * 3),
                ("crc_ok", C.c_uint8), ("ok_3of6", C.c_uint8), ("packet_rssi", C.c_uint32),
                ("current_rssi", C.c_uint32), ("serial", C.c_uint32), ("len", C.c_uint32),
                ("datagram", C.c_uint8 * 292)]


class WmbRepaired(C.Structure):
    """wmb_repaired (include/wmbus_b200_framer.h): one candidate's erasure repair"""
    _fields_ = [("outcome", C.c_int), ("erasures", C.c_uint32), ("blocks", C.c_uint32), ("had_line", C.c_uint32),
                ("line", WmbDecoded)]


# wmb_repaired.outcome
REP_NONE, REP_REPAIRED, REP_AMBIGUOUS, REP_TOO_MANY, REP_UNREPAIRABLE, REP_TRUNCATED = range(6)


class WmbRepairRecord(C.Structure):
    """wmb_repair_record (include/wmbus_b200_framer.h): the repair of one candidate of the streaming framer"""
    _fields_ = [("sync_sample", C.c_uint64), ("end_sample", C.c_uint64), ("chain", C.c_uint8), ("algo", C.c_uint8),
                ("soft_t1", C.c_uint8), ("soft_s1", C.c_uint8), ("reserved", C.c_uint8 * 4), ("repair", WmbRepaired)]

    @property
    def line(self):
        return self.repair.line


class WmbLineInfo(C.Structure):
    _fields_ = [("sync_sample", C.c_uint64), ("end_sample", C.c_uint64), ("chain", C.c_uint8), ("algo", C.c_uint8),
                ("crc_ok", C.c_uint8), ("valid", C.c_uint8), ("n", C.c_uint32), ("sum", C.c_int64),
                ("carrier_hz", C.c_double), ("offset_hz", C.c_double)]


# numpy mirror of wmb_line_info (one record per line; see include/wmbus_b200.h)
LINE_INFO_FIELDS = [("sync_sample", "<u8"), ("end_sample", "<u8"), ("chain", "u1"), ("algo", "u1"), ("crc_ok", "u1"),
                    ("valid", "u1"), ("n", "<u4"), ("sum", "<i8"), ("carrier_hz", "<f8"), ("offset_hz", "<f8")]


def line_info_dtype():
    import numpy as np
    return np.dtype(LINE_INFO_FIELDS)


# numpy mirror of wmb_burst (one record per burst piece; see include/wmbus_b200.h)
BURST_FIELDS = [("start_sample", "<u8"), ("end_sample", "<u8"), ("rssi_sum", "<u8"), ("sum", "<i8"),
                ("carrier_hz", "<f8"), ("offset_hz", "<f8"), ("n", "<u4"), ("chain", "u1"), ("peak", "u1"),
                ("valid", "u1"), ("flags", "u1")]
BURST_CONTINUED, BURST_CUT, BURST_AT_END = 1, 2, 4


def burst_dtype():
    import numpy as np
    return np.dtype(BURST_FIELDS)


# numpy mirror of wmb_snippet (one record per saved burst snippet; see include/wmbus_b200.h)
SNIPPET_FIELDS = [("start_sample", "<u8"), ("end_sample", "<u8"), ("start_iq", "<u8"), ("nbytes", "<u8"),
                  ("chain", "u1"), ("decoded", "u1"), ("flags", "u1"), ("lost", "u1"), ("pad", "<u4")]
SNIPPET_PRE, SNIPPET_POST = 2, 2          # WMB_SNIPPET_PRE / WMB_SNIPPET_POST: granules before / after a piece


def snippet_dtype():
    import numpy as np
    return np.dtype(SNIPPET_FIELDS)


# numpy mirror of wmb_telegram (one record per transmission; see include/wmbus_b200_framer.h)
TELEGRAM_FIELDS = [("sync_sample", "<u8"), ("id", "<u4"), ("m", "<u2"), ("len", "<u2"), ("failed", "<u4"),
                   ("chain", "u1"), ("decoded", "u1"), ("sources", "u1"), ("valid", "u1"), ("mode", "S3"),
                   ("manuf", "S4"), ("l", "u1"), ("c", "u1"), ("version", "u1"), ("type", "u1"), ("ci", "u1"),
                   ("pad", "u1", (4,))]
TLG_W = (128, 256)                        # WMB_TLG_W_T1C1, WMB_TLG_W_S1: decimated samples between matches of one group
TLG_T2A_LINE, TLG_RLA_LINE, TLG_T2A_REPAIR, TLG_RLA_REPAIR = 1, 2, 4, 8      # wmb_telegram.sources
TLG_F_L, TLG_F_C, TLG_F_M, TLG_F_ID, TLG_F_VERSION, TLG_F_TYPE, TLG_F_CI = 1, 2, 4, 8, 16, 32, 64   # wmb_telegram.valid


def telegram_dtype():
    import numpy as np
    return np.dtype(TELEGRAM_FIELDS)


def group_telegrams(lib, info, lines, repairs=()):
    """wmb_group_telegrams over line records (a numpy array of wmb_line_info), their decodes (a sequence of WmbDecoded,
    one per record) and repair records (WmbRepairRecord) -> (records, data): records a numpy array of wmb_telegram
    (telegram_dtype()), data a list with the datagram bytes of each record"""
    import numpy as np
    info = np.ascontiguousarray(info, dtype=line_info_dtype())
    assert len(info) == len(lines), "one decode per line record"
    dec = (WmbDecoded * max(len(lines), 1))(*lines)
    rep = (WmbRepairRecord * max(len(repairs), 1))(*repairs)
    cap = len(lines) + len(repairs)
    need = sum(int(d.len) for d, r in zip(lines, info) if r["crc_ok"]) + sum(int(r.repair.line.len) for r in repairs
                                                                           if r.repair.outcome == REP_REPAIRED)
    out = np.zeros(max(cap, 1), telegram_dtype())
    buf = np.zeros(max(need, 1), np.uint8)
    n = C.c_size_t(0)
    rc = lib.wmb_group_telegrams(info.ctypes.data if len(info) else None, dec, len(lines), rep, len(repairs),
                                 out.ctypes.data, cap, buf.ctypes.data, need, C.byref(n))
    if rc != 0:
        raise RuntimeError(f"wmb_group_telegrams failed ({rc})")
    out = out[:n.value]
    return out, _split(buf, out["len"])


def _split(buf, lens):
    """the concatenated datagrams in buf -> one bytes object per record"""
    import numpy as np
    ends = np.cumsum(lens, dtype=np.int64).tolist()
    raw = buf[:ends[-1] if ends else 0].tobytes()
    return [raw[a:b] for a, b in zip([0] + ends[:-1], ends)]


# numpy mirrors of wmb_line_quality and wmb_burst_quality (see include/wmbus_b200.h)
LINE_QUALITY_FIELDS = [("sync_sample", "<u8"), ("end_sample", "<u8"), ("n_hi", "<u4"), ("n_lo", "<u4"),
                       ("s1_hi", "<i8"), ("s1_lo", "<i8"), ("s2_hi", "<u8"), ("s2_lo", "<u8"), ("bits", "<u4"),
                       ("chain", "u1"), ("algo", "u1"), ("crc_ok", "u1"), ("valid", "u1"), ("deviation_hz", "<f8"),
                       ("eye_snr_db", "<f8"), ("chip_rate_hz", "<f8")]
BURST_QUALITY_FIELDS = [("start_sample", "<u8"), ("n_hi", "<u4"), ("n_lo", "<u4"), ("s1_hi", "<i8"), ("s1_lo", "<i8"),
                        ("s2_hi", "<u8"), ("s2_lo", "<u8"), ("deviation_hz", "<f8"), ("eye_snr_db", "<f8"),
                        ("chain", "u1"), ("valid", "u1"), ("pad", "V6")]


def line_quality_dtype():
    import numpy as np
    return np.dtype(LINE_QUALITY_FIELDS)


def burst_quality_dtype():
    import numpy as np
    return np.dtype(BURST_QUALITY_FIELDS)


# numpy mirror of wmb_spectrum_row (one record of the band survey; see include/wmbus_b200.h)
SPECTRUM_FIELDS = [("record", "<u8"), ("start_iq", "<u8"), ("blocks", "<u4"), ("bins", "<u4"), ("hz_low", "<f8"),
                   ("hz_step", "<f8")]


def spectrum_dtype():
    import numpy as np
    return np.dtype(SPECTRUM_FIELDS)


class WmbStats(C.Structure):
    _fields_ = [("input_samples", C.c_uint64), ("decimated_samples", C.c_uint64), ("batches", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("lanes_run", C.c_uint64), ("lanes_rerun", C.c_uint64),
                ("candidates", (C.c_uint64 * 2) * 2), ("lines", (C.c_uint64 * 2) * 2),
                ("lines_crc_ok", (C.c_uint64 * 2) * 2), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("demod_kernel_ms", C.c_double), ("bitsync_kernel_ms", C.c_double),
                ("batch_device_ms", C.c_double), ("rl_fallbacks", C.c_uint64), ("host_batch_ms", C.c_double),
                ("host_gather_ms", C.c_double), ("host_decode_ms", C.c_double), ("overflow_batches", C.c_uint64)]


def library_path() -> str:
    return os.path.join(PKG_DIR, LIB_NAME)


def build(verbose: bool = False) -> str:
    """Compile csrc/ for sm_90a into the in-tree libwmbus_b200.so and the rtl_wmbus_b200 CLI."""
    subprocess.run(["make", "-s", "-C", os.path.join(PKG_DIR, "csrc")] + ([] if not verbose else ["V=1"]), check=True)
    return library_path()


def _bind(lib):
    lib.wmb_default_opts.argtypes = [C.POINTER(WmbOpts)]
    lib.wmb_abi_version.restype = C.c_int
    lib.wmb_last_error.restype = C.c_char_p
    lib.wmb_version_string.restype = C.c_char_p
    lib.wmb_create.argtypes = [C.POINTER(WmbOpts), C.c_int, C.POINTER(C.c_void_p)]
    lib.wmb_destroy.argtypes = [C.c_void_p]
    lib.wmb_reset.argtypes = [C.c_void_p]
    lib.wmb_host_alloc.argtypes = [C.c_size_t]
    lib.wmb_host_alloc.restype = C.c_void_p
    lib.wmb_host_free.argtypes = [C.c_void_p]
    lib.wmb_push.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_push_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_poll.argtypes = [C.c_void_p, C.POINTER(WmbFrame), C.c_size_t, C.POINTER(C.c_size_t), C.c_int]
    lib.wmb_decode_frames.argtypes = [C.c_void_p, C.POINTER(WmbFrame), C.c_size_t]
    lib.wmb_take_lines.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int]
    lib.wmb_take_lines.restype = C.c_size_t
    lib.wmb_take_lines_info.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int, C.c_void_p,
                                        C.c_size_t]
    lib.wmb_take_lines_info.restype = C.c_size_t
    lib.wmb_process.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_char_p, C.c_size_t,
                                C.POINTER(C.c_size_t), C.c_int]
    lib.wmb_process.restype = C.c_long
    lib.wmb_process_device.argtypes = lib.wmb_process.argtypes
    lib.wmb_process_device.restype = C.c_long
    lib.wmb_get_stats.argtypes = [C.c_void_p, C.POINTER(WmbStats)]
    lib.wmb_debug_copy_stage.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_debug_copy_stage.restype = C.c_long
    lib.wmb_debug_copy_bits.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.wmb_debug_copy_bits.restype = C.c_long
    lib.wmb_debug_copy_events.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    lib.wmb_debug_copy_events.restype = C.c_long
    lib.wmb_debug_arith.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_seek.argtypes = [C.c_void_p, C.c_uint64]
    lib.wmb_set_line_window.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    lib.wmb_set_receiver.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32]
    lib.wmb_set_bursts.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    lib.wmb_take_bursts.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_set_line_quality.argtypes = [C.c_void_p, C.c_int]
    lib.wmb_set_snippets.argtypes = [C.c_void_p, C.c_int]
    lib.wmb_take_snippets.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_set_telegrams.argtypes = [C.c_void_p, C.c_int]
    lib.wmb_take_telegrams.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_group_telegrams.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                        C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_take_lines_quality.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int,
                                           C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_take_lines_quality.restype = C.c_size_t
    lib.wmb_take_bursts_quality.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_set_spectrum.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    lib.wmb_take_spectrum.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_debug_spectrum_tables.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
    lib.wmb_boundary_state.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.wmb_boundary_state.restype = C.c_long
    lib.wmb_pending_before.argtypes = [C.c_void_p, C.c_uint64]
    lib.wmb_pending_before.restype = C.c_long
    lib.wmb_frame_repair.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    lib.wmb_frame_repair_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.wmb_set_repair.argtypes = [C.c_void_p, C.c_uint32]
    lib.wmb_take_repairs.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.wmb_set_soft_bits.argtypes = [C.c_void_p, C.c_int]
    lib.wmb_set_repair_soft.argtypes = [C.c_void_p, C.c_uint32]
    lib.wmb_set_repair_t1_soft.argtypes = [C.c_void_p, C.c_uint32]
    lib.wmb_set_repair_s1_soft.argtypes = [C.c_void_p, C.c_uint32]
    lib.wmb_set_soft_bits_s1.argtypes = [C.c_void_p, C.c_int]
    lib.wmb_frame_repair_s1_soft.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.wmb_frame_repair_s1_soft_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32,
                                                    C.c_uint32, C.c_void_p]
    lib.wmb_frame_repair_t1_soft.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.wmb_frame_repair_t1_soft_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32,
                                                    C.c_uint32, C.c_void_p]
    lib.wmb_frame_soft.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.POINTER(C.c_int16))]
    lib.wmb_frame_repair_soft.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.wmb_frame_repair_soft_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                                 C.c_void_p]
    return lib


EXPORTS = ["wmb_reset", "wmb_host_alloc", "wmb_host_free", "wmb_default_opts", "wmb_abi_version", "wmb_last_error", "wmb_version_string", "wmb_create",
           "wmb_destroy", "wmb_push", "wmb_push_device", "wmb_poll", "wmb_decode_frames", "wmb_take_lines",
           "wmb_process", "wmb_process_device", "wmb_get_stats", "wmb_debug_copy_stage", "wmb_debug_copy_bits", "wmb_debug_copy_events", "wmb_debug_arith",
           "wmb_seek", "wmb_set_line_window", "wmb_boundary_state", "wmb_pending_before", "wmb_set_receiver",
           "wmb_take_lines_info", "wmb_set_bursts", "wmb_take_bursts", "wmb_set_spectrum", "wmb_take_spectrum",
           "wmb_debug_spectrum_tables", "wmb_set_line_quality", "wmb_take_lines_quality", "wmb_take_bursts_quality",
           "wmb_set_snippets", "wmb_take_snippets", "wmb_set_telegrams", "wmb_take_telegrams", "wmb_group_telegrams"]


def load_library(path: str | None = None):
    """dlopen libwmbus_b200.so.  Raises when it is missing: there is no fallback."""
    path = path or library_path()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: build it with __graft_entry__.build() "
                           f"(nvcc, sm_90a); rtl-wmbus_b200 has no CPU fallback")
    return _bind(C.CDLL(path))


def opts_from_flags(lib, flags: str = "", **kw) -> WmbOpts:
    """Build wmb_opts from a reference-style flag string, e.g. '-d 3 -s -o -v'."""
    o = WmbOpts()
    lib.wmb_default_opts(C.byref(o))
    toks = flags.split()
    i = 0
    while i < len(toks):
        t = toks[i]
        if t == "-o": o.remove_dc = 1
        elif t == "-a": o.accurate_atan = 0
        elif t == "-s": o.simultaneous = 1
        elif t == "-v": o.show_algorithm = 1
        elif t == "-f": pass
        elif t == "-d": i += 1; o.decimation = int(toks[i])
        elif t == "-r": i += 1; o.rla_enabled = 0 if toks[i] == "0" else 1
        elif t == "-t": i += 1; o.t2_enabled = 0 if toks[i] == "0" else 1
        elif t == "-p":
            i += 1
            if toks[i] in ("T", "t"): o.t1c1_enabled = 0
            elif toks[i] in ("S", "s"): o.s1_enabled = 0
            else: raise ValueError(toks[i])
        else:
            raise ValueError(f"unknown flag {t}")
        i += 1
    for k, v in kw.items():
        setattr(o, k, v)
    return o


class WmbusB200:
    """One decoding context (== one rtl_wmbus process) on one GPU.
    clock_lock=(t1c1, s1), access_code_errors=(t1c1, s1): receiver settings, see wmb_set_receiver() (default (2, 2) and
    (0, 0), the reference's).  They survive reset() and seek().
    burst_level=(t1c1, s1): the burst report's level per chain, see wmb_set_bursts() (0: off, the default); it survives
    reset() and seek() too.  take_bursts() hands out the closed pieces.
    spectrum=(bins, blocks_per_record): the band survey, see wmb_set_spectrum() (None: off, the default); it survives
    reset() and seek().  take_spectrum() hands out the closed records.
    quality=True: the signal-quality report, see wmb_set_line_quality() (off by default); it survives reset() and
    seek().  take_lines(quality=True) and take_bursts(quality=True) hand out its records.
    repair=e_max (1..3): erasure repair of the framer's T1 / S1 candidates, see wmb_set_repair() (0: off, the default);
    it survives reset() and seek().  take_repairs() hands out its records.
    repair_soft=k_max (1..6): with repair on, the C1 candidates are repaired from the soft values of their bits, see
    wmb_set_repair_soft() (0: off, the default); it survives reset() and seek().
    repair_t1_soft=s_max (1..6): with repair on, the T1 candidates that erasure repair gives up on are repaired from the
    soft values of their chips, see wmb_set_repair_t1_soft() (0: off, the default); it survives reset() and seek().
    repair_s1_soft=s_max (1..6): with repair on, the S1 candidates that erasure repair gives up on are repaired from the
    soft values of their chips, see wmb_set_repair_s1_soft() (0: off, the default); it survives reset() and seek().
    soft_bits=True (manual_frames=1 only): the soft value of every T1/C1 bit, see wmb_set_soft_bits() (off by default); it
    survives reset() and seek().  frame_soft() returns a polled frame's values and repair_frames(k_max=...) uses them.
    soft_bits_s1=True (manual_frames=1 only): the soft value of every S1 chip too, see wmb_set_soft_bits_s1().
    snippets=mode: the raw bytes around each burst piece, see wmb_set_snippets() (0: off, the default; 1: every piece;
    2: the pieces that did not decode); needs burst_level on a chain.  It survives reset() and seek().  take_snippets()
    hands them out.
    telegrams=True: one record per transmission from both bit syncs and the repairs, see wmb_set_telegrams() (off by
    default); it survives reset() and seek().  take_telegrams() hands out the final ones."""

    def __init__(self, flags: str = "", device: int = 0, lib=None, clock_lock=None, access_code_errors=None,
                 burst_level=None, spectrum=None, quality=False, repair=0, repair_soft=0, soft_bits=False,
                 repair_t1_soft=0, repair_s1_soft=0, soft_bits_s1=False, snippets=0, telegrams=False, **tuning):
        self.lib = lib or load_library()
        self.opts = opts_from_flags(self.lib, flags, **tuning)
        self._ctx = C.c_void_p()
        rc = self.lib.wmb_create(C.byref(self.opts), device, C.byref(self._ctx))
        if rc != 0:
            raise RuntimeError(f"wmb_create failed ({rc}): {self.lib.wmb_last_error().decode()}")
        self._out = C.create_string_buffer(1 << 22)
        if clock_lock is not None or access_code_errors is not None:
            lock = clock_lock if clock_lock is not None else (2, 2)
            errs = access_code_errors if access_code_errors is not None else (0, 0)
            try:
                for chain in (0, 1):
                    self.set_receiver(chain, lock[chain], errs[chain])
            except Exception:
                self.close()
                raise
        if burst_level is not None:
            try:
                for chain in (0, 1):
                    self.set_bursts(chain, burst_level[chain])
            except Exception:
                self.close()
                raise
        if spectrum is not None:
            try:
                self.set_spectrum(*spectrum)
            except Exception:
                self.close()
                raise
        if quality:
            try:
                self.set_line_quality(True)
            except Exception:
                self.close()
                raise
        if repair:
            try:
                self.set_repair(repair)
            except Exception:
                self.close()
                raise
        if repair_soft:
            try:
                self.set_repair_soft(repair_soft)
            except Exception:
                self.close()
                raise
        if repair_t1_soft:
            try:
                self.set_repair_t1_soft(repair_t1_soft)
            except Exception:
                self.close()
                raise
        if repair_s1_soft:
            try:
                self.set_repair_s1_soft(repair_s1_soft)
            except Exception:
                self.close()
                raise
        if soft_bits_s1:
            try:
                self.set_soft_bits_s1(True)
            except Exception:
                self.close()
                raise
        if soft_bits:
            try:
                self.set_soft_bits(True)
            except Exception:
                self.close()
                raise
        if snippets:
            try:
                self.set_snippets(snippets)
            except Exception:
                self.close()
                raise
        if telegrams:
            try:
                self.set_telegrams(True)
            except Exception:
                self.close()
                raise

    def close(self):
        if self._ctx:
            self.lib.wmb_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __enter__(self): return self
    def __exit__(self, *a): self.close()
    def __del__(self):
        try: self.close()
        except Exception: pass

    def _check(self, rc):
        if rc < 0:
            raise RuntimeError(f"libwmbus_b200 error {rc}: {self.lib.wmb_last_error().decode()}")
        return rc

    def _lines(self, n):
        if n <= 0:
            return []
        txt = C.string_at(self._out, n).decode("ascii")      # (.raw would copy the whole 4 MiB buffer)
        return txt.split("\n")[:-1] if txt.endswith("\n") else [l for l in txt.split("\n") if l]

    def _drain(self, taken, timestamp_mode):
        """wmb_process* hands out only the lines that fit the buffer; the rest stay queued -- fetch them too"""
        return self.take_lines(timestamp_mode) if taken else []

    def process(self, host_ptr, nbytes, flush=True, timestamp_mode=1, raw=False, info=False):
        """host_ptr: int address / ctypes pointer of cu8 bytes in host memory.
        info=True: (lines, records), records a numpy structured array of wmb_line_info (line_info_dtype()), one per line"""
        nl = C.c_size_t(0)
        if info:                                            # nothing taken by the call itself: every line gets its record
            self._check(self.lib.wmb_process(self._ctx, host_ptr, nbytes, int(flush), self._out, 0, C.byref(nl),
                                             timestamp_mode))
            return self.take_lines(timestamp_mode, info=True)
        n = self._check(self.lib.wmb_process(self._ctx, host_ptr, nbytes, int(flush), self._out,
                                             len(self._out), C.byref(nl), timestamp_mode))
        if raw:
            return self._raw(n, nl.value, timestamp_mode)
        return self._lines(n) + self._drain(nl.value, timestamp_mode)

    def process_bytes(self, data: bytes, flush=True, timestamp_mode=1, info=False):
        buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
        return self.process(C.cast(buf, C.c_void_p), len(data), flush, timestamp_mode, info=info)

    def process_device(self, dev_ptr: int, nbytes: int, flush=True, timestamp_mode=1, raw=False, info=False):
        """raw=True: the text exactly as the C ABI hands it out (bytes, one line per datagram), not a list of str
        info=True: (lines, records) as in process()"""
        nl = C.c_size_t(0)
        if info:
            self._check(self.lib.wmb_process_device(self._ctx, C.c_void_p(dev_ptr), nbytes, int(flush), self._out, 0,
                                                    C.byref(nl), timestamp_mode))
            return self.take_lines(timestamp_mode, info=True)
        n = self._check(self.lib.wmb_process_device(self._ctx, C.c_void_p(dev_ptr), nbytes, int(flush),
                                                    self._out, len(self._out), C.byref(nl), timestamp_mode))
        if raw:
            return self._raw(n, nl.value, timestamp_mode)
        return self._lines(n) + self._drain(nl.value, timestamp_mode)

    def _raw(self, n, taken, timestamp_mode):
        txt = C.string_at(self._out, n) if n > 0 else b""
        while taken:                                        # more lines than the buffer holds: fetch the rest
            k = C.c_size_t(0)
            m = self.lib.wmb_take_lines(self._ctx, self._out, len(self._out), C.byref(k), timestamp_mode)
            taken = k.value
            if taken:
                txt += C.string_at(self._out, m)
        return txt

    @staticmethod
    def split_lines(txt: bytes):
        return txt.decode("ascii").split("\n")[:-1] if txt else []

    def push(self, host_ptr, nbytes):
        self._check(self.lib.wmb_push(self._ctx, host_ptr, nbytes))

    def push_device(self, dev_ptr: int, nbytes: int):
        self._check(self.lib.wmb_push_device(self._ctx, dev_ptr, nbytes))

    def push_bytes(self, data: bytes):
        buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
        self.push(C.cast(buf, C.c_void_p), len(data))

    def poll(self, flush=False, cap=1 << 16):
        arr = (WmbFrame * cap)()
        n = C.c_size_t(0)
        self._check(self.lib.wmb_poll(self._ctx, arr, cap, C.byref(n), int(flush)))
        return arr, n.value

    def poll_flush(self):
        """end of input: process what is buffered and finish the telegrams in flight (lines stay queued)"""
        n = C.c_size_t(0)
        self._check(self.lib.wmb_poll(self._ctx, None, 0, C.byref(n), 1))

    def decode_frames(self, arr, n):
        self._check(self.lib.wmb_decode_frames(self._ctx, arr, n))

    def repair_frames(self, arr, n, e_max=2, device=True, k_max=0, soft=None, s_max=0, s1_max=0):
        """Erasure repair (wmb_frame_repair_device, or the host twin wmb_frame_repair with device=False) of the first n
        frames of arr, e.g. what poll() returned with manual_frames=1.  Returns an array of n WmbRepaired; lines of the
        repaired ones format with repaired_line().
        k_max (1..6): C1 soft repair too (wmb_frame_repair_soft_device / wmb_frame_repair_soft), with soft[i] the int16
        soft values of frame i (None: none); soft=None takes frame_soft() of every frame.
        s_max (1..6): T1 soft repair instead (wmb_frame_repair_t1_soft_device / wmb_frame_repair_t1_soft), with the same
        soft; s1_max (1..6): S1 soft repair instead (wmb_frame_repair_s1_soft_device / wmb_frame_repair_s1_soft).  At most
        one of k_max, s_max and s1_max can be given."""
        out = (WmbRepaired * max(n, 1))()
        if sum(1 for x in (k_max, s_max, s1_max) if x) > 1:
            raise ValueError("repair_frames: k_max (C1), s_max (T1) and s1_max (S1) are separate rules; give one of them")
        if k_max or s_max or s1_max:
            import numpy as np
            if soft is None:
                soft = [self.frame_soft(arr[i]) for i in range(n)]
            soft = [None if v is None else np.ascontiguousarray(v, np.int16) for v in soft]
            ptrs = (C.c_void_p * max(n, 1))(*[None if v is None else v.ctypes.data for v in soft[:n]])
            dev, host = ((self.lib.wmb_frame_repair_soft_device, self.lib.wmb_frame_repair_soft) if k_max else
                         (self.lib.wmb_frame_repair_t1_soft_device, self.lib.wmb_frame_repair_t1_soft) if s_max else
                         (self.lib.wmb_frame_repair_s1_soft_device, self.lib.wmb_frame_repair_s1_soft))
            kk = k_max or s_max or s1_max
            if device:
                self._check(dev(self._ctx, C.addressof(arr), ptrs, n, e_max, kk, C.addressof(out)))
            else:
                for i in range(n):
                    self._check(host(C.addressof(arr[i]), ptrs[i], e_max, kk, C.addressof(out[i])))
            return out
        if device:
            self._check(self.lib.wmb_frame_repair_device(self._ctx, C.addressof(arr), n, e_max, C.addressof(out)))
        else:
            for i in range(n):
                self._check(self.lib.wmb_frame_repair(C.addressof(arr[i]), e_max, C.addressof(out[i])))
        return out

    def repaired_line(self, r, algo_prefix=b"", timestamp=b"TS"):
        """the line of a repaired frame (a WmbRepaired, or a WmbRepairRecord of take_repairs()) in the stdout format
        (without its newline)"""
        fmt = C.CFUNCTYPE(C.c_size_t, C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t)(("wmb_format_line",
                                                                                                  self.lib))
        buf = C.create_string_buffer(2048)
        k = fmt(C.addressof(r.line), algo_prefix, timestamp, buf, 2048)
        return buf.raw[:k].decode().rstrip("\n")

    def take_lines(self, timestamp_mode=1, info=False, quality=False):
        """info=True: (lines, records), records a numpy structured array of wmb_line_info, one per line.
        quality=True: (lines, quality) with a numpy structured array of wmb_line_quality (line_quality_dtype()), one per
        line; with both: (lines, records, quality)"""
        nl = C.c_size_t(0)
        out = []
        if quality:
            import numpy as np
            cap = 1 << 14
            infos, quals = [], []
            while True:
                r = np.zeros(cap, line_info_dtype())
                q = np.zeros(cap, line_quality_dtype())
                n = self.lib.wmb_take_lines_quality(self._ctx, self._out, len(self._out), C.byref(nl), timestamp_mode,
                                                    r.ctypes.data, q.ctypes.data, cap)
                if not nl.value:
                    break
                out += self._lines(n)
                infos.append(r[:nl.value])
                quals.append(q[:nl.value])
            infos = np.concatenate(infos) if infos else np.zeros(0, line_info_dtype())
            quals = np.concatenate(quals) if quals else np.zeros(0, line_quality_dtype())
            return (out, infos, quals) if info else (out, quals)
        if not info:
            while True:
                n = self.lib.wmb_take_lines(self._ctx, self._out, len(self._out), C.byref(nl), timestamp_mode)
                if not nl.value:
                    break
                out += self._lines(n)
            return out
        import numpy as np
        cap = 1 << 14
        recs = []
        while True:
            r = np.zeros(cap, line_info_dtype())
            n = self.lib.wmb_take_lines_info(self._ctx, self._out, len(self._out), C.byref(nl), timestamp_mode,
                                             r.ctypes.data, cap)
            if not nl.value:
                break
            out += self._lines(n)
            recs.append(r[:nl.value])
        return out, (np.concatenate(recs) if recs else np.zeros(0, line_info_dtype()))

    def reset(self):
        self._check(self.lib.wmb_reset(self._ctx))

    def seek(self, first_iq_sample: int):
        """reset + position the stream at an absolute IQ sample of the capture (time-chunk sharding)"""
        self._check(self.lib.wmb_seek(self._ctx, first_iq_sample))

    def set_receiver(self, chain: int, clock_lock: int, access_code_errors: int):
        """clock-lock threshold and access-code bit errors of one chain (before the first push, or after reset/seek)"""
        self._check(self.lib.wmb_set_receiver(self._ctx, chain, clock_lock, access_code_errors))

    def set_bursts(self, chain: int, level: int):
        """burst report level of one chain, 0 = off (before the first push, or after reset/seek)"""
        self._check(self.lib.wmb_set_bursts(self._ctx, chain, level))

    def take_bursts(self, quality=False):
        """the closed burst pieces not taken yet, ordered by (start_sample, chain): a numpy structured array of
        wmb_burst (burst_dtype()); quality=True: (bursts, quality), quality the wmb_burst_quality records
        (burst_quality_dtype()), one per burst"""
        import numpy as np
        cap = 1 << 14
        parts, qparts = [], []
        while True:
            r = np.zeros(cap, burst_dtype())
            q = np.zeros(cap if quality else 0, burst_quality_dtype())
            n = C.c_size_t(0)
            self._check(self.lib.wmb_take_bursts_quality(self._ctx, r.ctypes.data, q.ctypes.data if quality else None,
                                                         cap, C.byref(n)))
            if n.value:
                parts.append(r[:n.value])
                qparts.append(q[:n.value])
            if n.value < cap:
                break
        b = np.concatenate(parts) if parts else np.zeros(0, burst_dtype())
        if not quality:
            return b
        return b, (np.concatenate(qparts) if qparts else np.zeros(0, burst_quality_dtype()))

    def set_snippets(self, mode: int):
        """0: off, 1: every burst piece, 2: the pieces that did not decode (before the first push, or after reset/seek)"""
        self._check(self.lib.wmb_set_snippets(self._ctx, mode))

    def take_snippets(self, cap=1 << 12, bytes_cap=64 << 20):
        """the snippets ready, in burst order: (records, data), records a numpy structured array of wmb_snippet
        (snippet_dtype()) and data a list with one bytes object per record.  bytes_cap holds any one snippet: a piece
        spans at most 2^17 + 2^16 samples, its snippet at most 101 granules of 4096 d bytes (10 MB at d = 25)"""
        import numpy as np
        recs, data = [], []
        buf = np.zeros(bytes_cap, np.uint8)
        while True:
            r = np.zeros(cap, snippet_dtype())
            n = C.c_size_t(0)
            self._check(self.lib.wmb_take_snippets(self._ctx, r.ctypes.data, cap, buf.ctypes.data, bytes_cap, C.byref(n)))
            if n.value == 0:
                break
            r = r[:n.value]
            at = 0
            for x in r:
                data.append(buf[at:at + int(x["nbytes"])].tobytes())
                at += int(x["nbytes"])
            recs.append(r)
        return (np.concatenate(recs) if recs else np.zeros(0, snippet_dtype())), data

    def set_telegrams(self, on: bool):
        """telegram records on / off (before the first push, or after reset/seek; not with manual_frames)"""
        self._check(self.lib.wmb_set_telegrams(self._ctx, 1 if on else 0))

    def take_telegrams(self, cap=1 << 12):
        """the final telegram records, in order: (records, data), records a numpy structured array of wmb_telegram
        (telegram_dtype()) and data a list with the datagram bytes of each record"""
        import numpy as np
        recs, data = [], []
        buf = np.zeros(cap * 292, np.uint8)          # any cap records' datagrams fit
        while True:
            r = np.zeros(cap, telegram_dtype())
            n = C.c_size_t(0)
            self._check(self.lib.wmb_take_telegrams(self._ctx, r.ctypes.data, cap, buf.ctypes.data, len(buf), C.byref(n)))
            if n.value == 0:
                break
            r = r[:n.value]
            data += _split(buf, r["len"])
            recs.append(r)
        return (np.concatenate(recs) if recs else np.zeros(0, telegram_dtype())), data

    def set_line_quality(self, on: bool):
        """signal-quality report on / off (before the first push, or after reset/seek)"""
        self._check(self.lib.wmb_set_line_quality(self._ctx, 1 if on else 0))

    def set_repair_soft(self, k_max: int):
        """C1 soft repair of the streaming framer's candidates, k_max 1..6 (0 = off; before the first push, or after reset()
        / seek()); it acts while set_repair() has repair on"""
        self._check(self.lib.wmb_set_repair_soft(self._ctx, k_max))

    def set_repair_t1_soft(self, s_max: int):
        """T1 soft repair of the streaming framer's candidates, s_max 1..6 (0 = off; before the first push, or after
        reset() / seek()); it acts while set_repair() has repair on"""
        self._check(self.lib.wmb_set_repair_t1_soft(self._ctx, s_max))

    def set_repair_s1_soft(self, s_max: int):
        """S1 soft repair of the streaming framer's candidates, s_max 1..6 (0 = off; before the first push, or after
        reset() / seek()); it acts while set_repair() has repair on"""
        self._check(self.lib.wmb_set_repair_s1_soft(self._ctx, s_max))

    def set_soft_bits_s1(self, on: bool):
        """soft values of the S1 chips (manual_frames=1; before the first push, or after reset() / seek())"""
        self._check(self.lib.wmb_set_soft_bits_s1(self._ctx, int(bool(on))))

    def set_soft_bits(self, on: bool):
        """soft values of the T1/C1 bits (before the first push, or after reset() / seek())"""
        self._check(self.lib.wmb_set_soft_bits(self._ctx, int(bool(on))))

    def frame_soft(self, frame):
        """the int16 soft values of a frame of the last poll(), parallel to its bits (a copy); None for S1 frames
        (unless soft_bits_s1 is on) or when soft values are off"""
        import numpy as np
        p = C.POINTER(C.c_int16)()
        self._check(self.lib.wmb_frame_soft(self._ctx, C.addressof(frame), C.byref(p)))
        if not p:
            return None
        return np.ctypeslib.as_array(p, (frame.nbits,)).copy()

    def set_repair(self, e_max: int):
        """erasure repair of the streaming framer's candidates, e_max 1..3 (0 = off; before the first push, or after
        reset/seek)"""
        self._check(self.lib.wmb_set_repair(self._ctx, e_max))

    def take_repairs(self, cap=1 << 12):
        """the repair records not taken yet, in (end_sample, chain * 2 + (algo == t2a), sync_sample) order: a list of
        WmbRepairRecord; the lines of the REPAIRED ones format with repaired_line()"""
        out = []
        while True:
            arr = (WmbRepairRecord * cap)()
            n = C.c_size_t(0)
            self._check(self.lib.wmb_take_repairs(self._ctx, arr, cap, C.byref(n)))
            out += list(arr[:n.value])
            if n.value < cap:
                return out

    def set_spectrum(self, bins: int, blocks_per_record: int):
        """band survey: bins 256 .. 2048 (0 = off), blocks per record (before the first push, or after reset/seek)"""
        self._check(self.lib.wmb_set_spectrum(self._ctx, bins, blocks_per_record))
        self._spec_bins = bins

    def take_spectrum(self):
        """the closed survey records not taken yet, in record order: (rows, sum, peak) -- rows a numpy structured array
        of wmb_spectrum_row (spectrum_dtype()), sum a [n, bins] uint64 array, peak a [n, bins] float32 array"""
        import numpy as np
        cap = 256                                           # rows per call; sum / peak sized for the largest N
        rows, sums, peaks = [], [], []
        while True:
            r = np.zeros(cap, spectrum_dtype())
            s = np.zeros((cap, 2048), np.uint64)
            p = np.zeros((cap, 2048), np.float32)
            n = C.c_size_t(0)
            self._check(self.lib.wmb_take_spectrum(self._ctx, r.ctypes.data, s.ctypes.data, p.ctypes.data, cap,
                                                   C.byref(n)))
            k = n.value
            if k:
                nb = int(r["bins"][0])
                rows.append(r[:k])
                sums.append(s.reshape(-1)[:k * nb].reshape(k, nb))
                peaks.append(p.reshape(-1)[:k * nb].reshape(k, nb))
            if k < cap:
                break
        if not rows:
            nb = getattr(self, "_spec_bins", 0)              # (no record: [0, bins] arrays, so parts concatenate)
            return np.zeros(0, spectrum_dtype()), np.zeros((0, nb), np.uint64), np.zeros((0, nb), np.float32)
        return np.concatenate(rows), np.concatenate(sums), np.concatenate(peaks)

    def set_line_window(self, sync_lo: int, sync_hi: int):
        self._check(self.lib.wmb_set_line_window(self._ctx, sync_lo, sync_hi))

    def pending_before(self, sync_hi: int) -> int:
        """telegrams in flight whose access-code match lies below decimated sample sync_hi"""
        return self._check(self.lib.wmb_pending_before(self._ctx, sync_hi))

    def boundary_state(self) -> bytes:
        if not hasattr(self, "_bbuf"):
            self._bbuf = C.create_string_buffer(1 << 22)        # (allocating and copying 4 MiB per call cost 2 ms)
        n = self._check(self.lib.wmb_boundary_state(self._ctx, self._bbuf, len(self._bbuf)))
        return C.string_at(self._bbuf, n)

    def stats(self) -> WmbStats:
        s = WmbStats()
        self._check(self.lib.wmb_get_stats(self._ctx, C.byref(s)))
        return s

    def debug_stage(self, chain: int, n: int):
        import numpy as np
        dphi = np.zeros(n, np.float32)
        rssi = np.zeros(n, np.uint8)
        got = self._check(self.lib.wmb_debug_copy_stage(self._ctx, chain, dphi.ctypes.data, rssi.ctypes.data, n))
        return dphi[:got], rssi[:got]

    def debug_bits(self, chain: int, which: int, n: int):
        """Unpacked 0/1 array of the last batch's data bits (0), time2 strobes (1) or clock signs (2)."""
        import numpy as np
        words = np.zeros((n + 31) // 32, np.uint32)
        got = self._check(self.lib.wmb_debug_copy_bits(self._ctx, chain, which, words.ctypes.data, len(words)))
        return np.unpackbits(words[:got].view(np.uint8), bitorder="little")[:n]

    def debug_events(self, chain: int, algo: int, cap: int = 1 << 22):
        """The last batch's bit events of one stream as (sample, rssi, reset, sync, bit) arrays."""
        import numpy as np
        ev = np.zeros(cap, np.uint64)
        got = self._check(self.lib.wmb_debug_copy_events(self._ctx, chain, algo, ev.ctypes.data, cap))
        ev = ev[:got]
        return dict(m=ev >> np.uint64(24), rssi=(ev >> np.uint64(16)) & np.uint64(0xFF), reset=(ev >> np.uint64(2)) & np.uint64(1),
                    sync=(ev >> np.uint64(1)) & np.uint64(1), bit=ev & np.uint64(1))

    def debug_arith(self, mode: int, y, x):
        """device arithmetic test hook: see wmb_debug_arith() in include/wmbus_b200.h"""
        import numpy as np
        y = np.ascontiguousarray(y, np.float32); x = np.ascontiguousarray(x, np.float32)
        out = np.zeros(len(y), np.float32)
        self._check(self.lib.wmb_debug_arith(self._ctx, mode, y.ctypes.data, x.ctypes.data, out.ctypes.data, len(y)))
        return out
