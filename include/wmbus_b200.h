/*
 * wmbus_b200.h -- C ABI of libwmbus_b200.so: the H100 (sm_90a) replacement for the
 * per-sample DSP hot path of rtl-wmbus (cu8 IQ -> box filter/decimate -> FM
 * discriminator -> FIR -> slicer/RSSI -> time2 + run-length bit sync -> access-code
 * correlation -> T1/C1/S1 framing -> datagram lines).
 *
 * The reference (xaelsouth/rtl-wmbus @ b6a7705) exposes no library interface: its
 * only boundary is the process contract of main() (rtl_wmbus.c:1217-1372: argv,
 * stdin cu8 in 4096-byte items, one stdout line per telegram).  The entry points
 * below are the seams a maintainer would cut when moving that loop onto a GPU; each
 * one cites the reference code it replaces.  Plain C types only -- no CUDA, torch or
 * C++ types cross this boundary.
 *
 * Threading: one caller per context (the reference is single-threaded and not
 * re-entrant: all filter state is function-local statics, e.g. rtl_wmbus.c:168-175).
 * Several contexts may live in one process (one per GPU / per capture).
 *
 * There is NO CPU fallback: wmb_create() fails with WMB_E_NODEVICE when no CUDA
 * device is usable.
 */
#ifndef WMBUS_B200_H
#define WMBUS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WMB_ABI_VERSION 2

/* error codes (negative) */
#define WMB_OK             0
#define WMB_E_INVAL       -1   /* bad argument / unsupported option value          */
#define WMB_E_NODEVICE    -2   /* no usable CUDA device (there is no CPU fallback) */
#define WMB_E_CUDA        -3   /* CUDA runtime error; see wmb_last_error()         */
#define WMB_E_NOMEM       -4
#define WMB_E_OVERFLOW    -5   /* internal event/frame buffer overflow (pathological input) */
#define WMB_E_STATE       -6   /* call order violated                               */

#define WMB_CHAIN_T1C1 0
#define WMB_CHAIN_S1   1
#define WMB_ALGO_RLA   0       /* run-length bit sync   (rtl_wmbus.c:617-803) */
#define WMB_ALGO_T2A   1       /* "time2" clock recovery (rtl_wmbus.c:806-852, :1080-1115) */

/* Options == the reference's command-line switches (rtl_wmbus.c:855-866, getopt
 * string "ofad:p:r:vVst:" at :896). */
typedef struct wmb_opts {
    uint32_t decimation;      /* -d N : input rate = N x 800 kS/s; default 2 (:857); N <= 25 (20 MS/s) */
    uint8_t  accurate_atan;   /* 0 with -a (cross-product discriminator, :536-551)         */
    uint8_t  remove_dc;       /* -o  (:497-515)                                            */
    uint8_t  rla_enabled;     /* 0 with -r 0                                               */
    uint8_t  t2_enabled;      /* 0 with -t 0                                               */
    uint8_t  t1c1_enabled;    /* 0 with -p T                                               */
    uint8_t  s1_enabled;      /* 0 with -p S                                               */
    uint8_t  simultaneous;    /* -s : +-325 kHz translation (:974-1031); 2: the same mixer with the carriers of
                                 carrier_25khz[] below (not a switch of the reference)       */
    uint8_t  show_algorithm;  /* -v : prefix lines with rla; / t2a;                        */
    /* tuning knobs (0 = library default); they never change results, only how the
     * work is cut up on the device */
    uint32_t chunk_samples;   /* decimated samples per bit-sync lane                       */
    uint32_t warmup_samples;  /* speculative warm-up before each lane                      */
    uint32_t max_batch_mib;   /* largest batch handed to the device at once (default 256)  */
    uint32_t manual_frames;   /* 1: wmb_push only gathers candidates; the caller drives the
                                 framers with wmb_poll + wmb_decode_frames.  0 (default):
                                 wmb_push feeds the context's framers itself.            */
    uint32_t reserved[2];     /* test knobs, 0 in production: [0] = 1 forces the monolithic run-length lanes for
                                 T1/C1; [1] bit 0 keeps the clock-sign words for wmb_debug_copy_bits(.., 2, ..),
                                 [1] bit 1 sizes the run-length streams' event rings by the large-batch rule (a
                                 quarter event per sample) also for small batches, [1] >> 8 (if not 0) is the size of
                                 the per-batch candidate tables: both to reach the overflow paths
                                 (wmb_stats.overflow_batches) with a small capture                                 */
    /* simultaneous == 2 (SURVEY 8f N3, many carriers per capture): offset of the carrier the T1/C1 chain [0] and the
     * S1 chain [1] listen to from the capture's centre frequency, in units of 25 kHz (the grid of the reference's
     * table, rtl_wmbus.c:974-993), |offset| <= fs / 2.  The reference's -s is {+13, -13}.  A capture with more than two
     * carriers is decoded by several contexts over the same input (shard.decode_carriers in the Python mirror). */
    int32_t  carrier_25khz[2];
    /* SURVEY 8f N4 -- one of the reference's dormant pre-decimation low-passes (rtl_wmbus.c:197-333, never called
     * upstream) takes the place of the moving averages in front of the decimation:
     *   1  lp_fir_butter_1600kHz_160kHz_200kHz_{t1_c1,s1}: 23-tap float FIR through firf() (fir.h:49-72)
     *   2  lp_ppf_butter_1600kHz_160kHz_200kHz: the same taps as a two-phase polyphase filter, ppf() (ppf.h:44-58)
     *   3  lp_firfp_butter_1600kHz_160kHz_200kHz: 1 in 24.8 fixed point, firfp() (fir.h:106-130, fixedptc.h)
     *   4  lp_ppffp_butter_1600kHz_160kHz_200kHz: 2 in 24.8 fixed point, ppffp() (ppf.h:69-83)
     * 1.6 MS/s only (decimation 2).  Not a switch of the reference: there are no reference lines to compare with; the
     * stages are checked against those functions themselves (oracle/ref_stages.c). */
    uint32_t prefilter;
} wmb_opts;

typedef struct wmb_ctx wmb_ctx;

/* One bit delivered to a framer, as produced on the device.  Bit layout of `w`:
 *   [31:9] sample offset (decimated samples) relative to wmb_frame.sync_sample
 *   [8:1]  (unsigned)rssi at that sample  (the `unsigned rssi` argument of
 *          t1_c1_packet_decoder(), t1_c1_packet_decoder.h:649)
 *   [0]    data bit                                                                */
typedef uint32_t wmb_bit;
#define WMB_BIT_DATA(w)   ((w) & 1u)
#define WMB_BIT_RSSI(w)   (((w) >> 1) & 0xFFu)
#define WMB_BIT_OFFSET(w) ((w) >> 9)

/* A framing candidate: the bit on which an access code matched (bits[0], the bit the
 * reference flags with PACKET_PREAMBLE_DETECTED, rtl_wmbus.c:773-776 / :822-825)
 * followed by the bits the same bit-sync instance produced after it.  For the
 * run-length algorithm the list stops where that algorithm reset itself (which also
 * resets its decoder, rtl_wmbus.c:717-726).                                         */
typedef struct wmb_frame {
    uint64_t sync_sample;     /* global decimated-sample index of bits[0]                 */
    uint64_t ordinal;         /* index of bits[0] in its (chain, algo) bit stream         */
    uint8_t  chain;           /* WMB_CHAIN_*                                              */
    uint8_t  algo;            /* WMB_ALGO_*                                               */
    uint8_t  truncated;       /* 1: the list ends before the header's length was reached    */
    uint8_t  reserved;        /* 1: partial -- the stream has not produced the remaining bits
                                 yet; the candidate is delivered again by a later poll     */
    uint32_t nbits;           /* number of entries in bits[] (>= 1)                       */
    const wmb_bit *bits;      /* owned by the context until the next wmb_push/wmb_poll    */
} wmb_frame;

/* ---- context ------------------------------------------------------------------ */

void        wmb_default_opts(wmb_opts *o);
int         wmb_abi_version(void);
const char *wmb_last_error(void);
const char *wmb_version_string(void);

/* Replaces the per-process set-up of main() (rtl_wmbus.c:1249-1296: algorithm
 * structs reset, chain/discriminator selection, mixer look-up tables). */
int  wmb_create(const wmb_opts *o, int cuda_device, wmb_ctx **out);
void wmb_destroy(wmb_ctx *c);
/* Start over with a new capture (same as destroy + create, without re-allocating). */
int  wmb_reset(wmb_ctx *c);

/* Receiver settings of one chain (WMB_CHAIN_*), for both of its algorithms -- the reference's two tuning constants
 * that it marks as future options:
 *   clock_lock          1..16, default 2: the time2 algorithm samples the data bit on the clock_lock-th clock sample
 *                       after a rising edge of the clock, i.e. on sample m iff the clock reads low at m-L-1 and high at
 *                       m-L..m (opts_CLOCK_LOCK_THRESHOLD_T1_C1 / _S1, rtl_wmbus.c:865-866, used at :1092-1111 and
 *                       :1184-1203).  Before the first sample the clock reads low.
 *   access_code_errors  default 0: a bit carries the access-code flag iff the shift register differs from the access
 *                       code in at most this many bits (ACCESS_CODE_T1_C1_ERRORS / ACCESS_CODE_S1_ERRORS, :99, :103,
 *                       compared at :688, :773, :822, :846).  At most 3 for T1/C1 (at 4 the preamble 0x5555 matches
 *                       0x543D) and 6 for S1.
 * Valid before the first push or right after wmb_reset / wmb_seek (else WMB_E_STATE); out-of-range values give
 * WMB_E_INVAL.  The settings survive wmb_reset and wmb_seek and are part of wmb_boundary_state(). */
int  wmb_set_receiver(wmb_ctx *c, int chain, uint32_t clock_lock, uint32_t access_code_errors);

/* Page-locked host memory for input buffers (the reference reads stdin into a 4096-byte
 * stack array, rtl_wmbus.c:1249; a GPU pipeline wants to DMA straight out of the read
 * buffer).  wmb_push() accepts any host pointer; pinned ones are copied asynchronously. */
void *wmb_host_alloc(size_t nbytes);
void  wmb_host_free(void *p);

/* ---- sample path (the hot loop, rtl_wmbus.c:1298-1357) ------------------------ */

/* Feed cu8 bytes from HOST memory.  Any length; the library consumes whole
 * 4096-byte items like the reference's fread (rtl_wmbus.c:1301) and keeps a
 * remainder for the next call.  Work is queued asynchronously (pinned staging ring,
 * H2D copy and kernels on the context's streams). */
int  wmb_push(wmb_ctx *c, const uint8_t *cu8, size_t nbytes);

/* Same, for bytes already resident in DEVICE memory of the context's GPU
 * (nbytes % 4096 == 0).  Used by the benchmark's device-resident leg. */
int  wmb_push_device(wmb_ctx *c, const void *dev_cu8, size_t nbytes);

/* Wait for queued work and hand out framing candidates in stream order per
 * (chain, algo).  flush != 0 declares end of input (the reference's EOF): pending
 * candidates are delivered truncated.  Returns the number of frames in *n. */
int  wmb_poll(wmb_ctx *c, wmb_frame *out, size_t cap, size_t *n, int flush);

/* ---- host-side framers (t1_c1_packet_decoder.h, s1_packet_decoder.h) ---------- */

/* Feed frames (as returned by wmb_poll, any interleaving of the four streams) to the
 * context's framers: 3-out-of-6 / NRZ / Manchester decode, L-field, RSSI abort,
 * block CRCs, CRC strip, line formatting -- the work of t1_c1_packet_decoder()
 * (t1_c1_packet_decoder.h:649-712) and s1_packet_decoder() (s1_packet_decoder.h:233-282).
 * Completed lines are appended to the context's line queue in the reference's output
 * order (finish sample, then T1/C1-rla, T1/C1-t2a, S1-rla, S1-t2a; rtl_wmbus.c:1074,
 * :1106, :1166, :1198). */
int  wmb_decode_frames(wmb_ctx *c, const wmb_frame *frames, size_t n);

/* Copy queued lines ('\n'-terminated, concatenated) into buf; returns the number of
 * bytes written (0 when none); *n_lines (optional) receives the line count.  Lines
 * that do not fit stay queued.  timestamp_mode: 0 = wall clock at delivery
 * (rtl_wmbus_util.h:10-39 format), 1 = the literal TS, 2 = the stream position at which the
 * reference would print the line, "@<decimated sample of the telegram's last bit>.<chain*2 + (algo == t2a)>":
 * sorting by it merges lines of several contexts (time-chunk sharding) into the reference's print order. */
size_t wmb_take_lines(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode);

/* What the receiver measured for one line, beside its text.  The carrier offset is the mean discriminator output over
 * 32 nominal chips of the telegram's preamble, in decimated samples (800 kS/s) before the access-code match s:
 * T1/C1 [s-384, s-128), S1 [s-1367, s-586), clipped to the samples pushed since the last wmb_reset / wmb_seek (n of
 * them are left).  sum = sum over that window of rint(dphi * 2^24), dphi the post-FIR, pre-DC-block discriminator
 * output (wmb_debug_copy_stage); exact, whatever the batch cut or thread order.
 *   offset_hz = sum / n / 2^24 * 400 kHz / G, G the DC gain (sum of taps) of the chain's post-demod FIR,
 * relative to carrier_hz, the carrier the chain listens to (0; +-325 kHz with -s; carrier_25khz[chain] * 25 kHz with
 * simultaneous = 2).  Positive: the telegram lies above that carrier.  valid = 0 (offset_hz NaN) when n = 0, with -a
 * (the cross-product discriminator is not a frequency), and for lines of frames handed to wmb_decode_frames. */
typedef struct wmb_line_info {
    uint64_t sync_sample;     /* decimated sample of the access-code match                                   */
    uint64_t end_sample;      /* decimated sample of the telegram's last bit                                 */
    uint8_t  chain;           /* WMB_CHAIN_*                                                                 */
    uint8_t  algo;            /* WMB_ALGO_*                                                                  */
    uint8_t  crc_ok;
    uint8_t  valid;
    uint32_t n;               /* samples in the window                                                      */
    int64_t  sum;             /* sum of rint(dphi * 2^24) over the window                                    */
    double   carrier_hz;
    double   offset_hz;
} wmb_line_info;

/* wmb_take_lines that also fills info[i] for the i-th line taken; it takes at most info_cap lines (info == NULL: no
 * records, no limit -- wmb_take_lines is this call).  Lines not taken stay queued. */
size_t wmb_take_lines_info(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode,
                           wmb_line_info *info, size_t info_cap);

/* ---- burst report: every signal burst on a chain, decoded or not ------------------------------------------------
 * Off by default.  wmb_set_bursts(ctx, chain, level) with level 1..255 turns it on for a chain.  On the chain's
 * (unsigned)rssi[m] (the scale of the PACKET_RSSI column; wmb_debug_copy_stage) and dphi[m], in decimated samples
 * (800 kS/s):
 *   1. above[m] = rssi[m] >= level.  Samples before the first one pushed since wmb_reset / wmb_seek are below.
 *   2. Bridge: a stretch of fewer than G below samples with an above sample on both sides counts as above.  This gives
 *      maximal runs [s, e), e one past the last above sample.
 *   3. Cut: a run is cut at every multiple of P = 2^16 (global decimated index) at least Q = 2^17 samples after its
 *      start s.  No telegram is that long, so none is cut; and a piece depends on at most Q + P + G earlier samples, so
 *      a time chunk with a 2^18-sample left halo reports the pieces of the sequential run.  A piece after a cut has
 *      WMB_BURST_CONTINUED, a piece ending at one WMB_BURST_CUT.
 *   4. Pieces of at least Lmin samples are reported, with peak = max rssi, rssi_sum = sum of rssi over [start, end),
 *      and the carrier offset as in wmb_line_info over the window [start + g0, min(end, start + g0 + w)) (n samples,
 *      sum = sum of rint(dphi * 2^24)): offset_hz = sum / n / 2^24 * 400 kHz / G_fir relative to carrier_hz.
 *      valid = 0 (offset_hz NaN) with -a or when n = 0.
 *   5. At end of input (flush) a run still open is closed one past its last above sample, WMB_BURST_AT_END.
 *              G (bridge)   Lmin   g0    w
 *     T1/C1    64           256    64    256      (8 chips, 32 chips, 8 chips, 32 chips)
 *     S1       196          782    196   781
 * A piece is handed out once it is closed and no piece still to come can start before it: wmb_take_bursts returns
 * them ordered by (start_sample, chain).  Join them with lines on sync_sample in [start_sample, end_sample) of the same
 * chain. */
#define WMB_BURST_CONTINUED 1u
#define WMB_BURST_CUT       2u
#define WMB_BURST_AT_END    4u

typedef struct wmb_burst {
    uint64_t start_sample;    /* decimated sample of the piece's first sample                                */
    uint64_t end_sample;      /* one past its last sample                                                    */
    uint64_t rssi_sum;        /* sum of (unsigned)rssi over [start_sample, end_sample)                       */
    int64_t  sum;             /* sum of rint(dphi * 2^24) over the offset window                             */
    double   carrier_hz;
    double   offset_hz;
    uint32_t n;               /* samples in the offset window                                                */
    uint8_t  chain;           /* WMB_CHAIN_*                                                                 */
    uint8_t  peak;            /* max (unsigned)rssi                                                          */
    uint8_t  valid;
    uint8_t  flags;           /* WMB_BURST_*                                                                 */
} wmb_burst;

/* level 0 (default): off; 1..255: on.  Valid before the first push or right after wmb_reset / wmb_seek (else
 * WMB_E_STATE); a bad chain or level > 255 gives WMB_E_INVAL.  The level survives wmb_reset and wmb_seek.  A chain
 * that the options turn off reports nothing. */
int wmb_set_bursts(wmb_ctx *c, int chain, uint32_t level);

/* Copy up to cap closed pieces into out, ordered by (start_sample, chain); *n receives their number.  Pieces not
 * taken stay queued. */
int wmb_take_bursts(wmb_ctx *c, wmb_burst *out, size_t cap, size_t *n);

/* ---- burst snippets: the raw cu8 bytes around each burst, replayable ----------------------------------------------
 * Off by default.  d is the decimation; a granule is 2048 decimated samples, 2048 d IQ samples, 4096 d bytes: granule g
 * covers decimated samples [2048 g, 2048 g + 2048), and its edges are the positions wmb_seek accepts.
 *   1. Which bursts: every piece wmb_take_bursts hands out (so snippets need wmb_set_bursts on at least one chain).
 *   2. Bounds: the snippet of a piece [s, e) covers the granules [lo, hi),
 *        lo = max(g_first, floor(s / 2048) - WMB_SNIPPET_PRE),  hi = min(ceil(e / 2048) + WMB_SNIPPET_POST, end),
 *      g_first the first granule pushed since wmb_reset / wmb_seek, end the end of the input consumed (at the end of
 *      input a last partial granule counts with the bytes consumed).  Its bytes are the input's bytes
 *      [lo 4096 d, hi 4096 d) relative to the capture (the index wmb_seek sets), as they were pushed.
 *   3. Decoded: the same chain has a line with CRC_OK = 1, or (repair on) a REPAIRED repair record, whose access-code
 *      match lies in [s, e) and in the line window.  A piece is handed out once it is closed, its last granule has
 *      been pushed (or the input ended), and no telegram of its chain matched in [s, e) is still in flight
 *      (wmb_pending_before's condition): so `decoded` is final.  Mode 1 hands out every piece, mode 2 only those that
 *      did not decode.
 *   4. Replay: pushing a snippet into a fresh context with the same options and receiver, repair and burst settings,
 *      after wmb_seek(start_iq), gives the lines of the full run (same text under timestamp_mode 1, same sync_sample)
 *      for every line whose match lies in [s, e); it may give more (its decoders start idle).  2048 d is a multiple of
 *      d and of the mixer's period, so the snippet pushed without a seek has the same decimation and mixer phases.
 *   5. Device memory: the kept granules of a batch go to a pool of at most 64 MiB per result slot (4 slots, and as
 *      much pinned host memory).  A snippet with a granule that did not fit is handed out with lost = 1 and no bytes,
 *      and wmb_stats.overflow_batches counts its batch. */
#define WMB_SNIPPET_PRE  2
#define WMB_SNIPPET_POST 2

typedef struct wmb_snippet {
    uint64_t start_sample;    /* the piece, as in wmb_burst                                                  */
    uint64_t end_sample;
    uint64_t start_iq;        /* lo 2048 d: the IQ sample of the snippet's first byte pair (for wmb_seek)      */
    uint64_t nbytes;          /* (hi - lo) 4096 d, less at the end of input; 0 when lost                      */
    uint8_t  chain;           /* WMB_CHAIN_*                                                                 */
    uint8_t  decoded;         /* 1: a CRC-ok or repaired telegram matched in the piece (point 3)              */
    uint8_t  flags;           /* WMB_BURST_*                                                                 */
    uint8_t  lost;            /* 1: a granule did not fit the device pool; no bytes                          */
    uint32_t pad;
} wmb_snippet;

/* mode 0: off (the default), 1: every burst piece, 2: the pieces that did not decode.  A mode outside 0..2 gives
 * WMB_E_INVAL (checked first); valid before the first push or right after wmb_reset / wmb_seek (else WMB_E_STATE).
 * The mode survives wmb_reset and wmb_seek.  The first push fails with WMB_E_STATE when snippets are on and no chain
 * has the burst report on. */
int wmb_set_snippets(wmb_ctx *c, int mode);

/* Copy whole snippets in the burst order (start_sample, chain): recs[i] and its nbytes bytes, concatenated in bytes.
 * Stops at cap records or when the next snippet's bytes do not fit bytes_cap; *n receives the number copied.  Snippets
 * not taken stay queued. */
int wmb_take_snippets(wmb_ctx *c, wmb_snippet *recs, size_t cap, uint8_t *bytes, size_t bytes_cap, size_t *n);

/* ---- signal quality: FSK deviation, eye SNR and chip rate of each line and burst --------------------------------
 * Off by default; wmb_set_line_quality(ctx, 1) turns it on.  Over the carrier-offset window [lo, hi) of a line
 * (wmb_line_info: T1/C1 [s-384, s-128), S1 [s-1367, s-586), clipped) or of a burst (wmb_burst: [start + g0,
 * min(end, start + g0 + w))), n samples, x[q] = rint(dphi[q] * 2^24), sum = sum of x:
 *   1. Class: sample q is high iff x[q] n >= sum (the window mean, in int64, no division), else low.  A sample q in
 *      [lo + 1, hi - 1) counts iff q - 1, q and q + 1 are all of the same class: the FIR's chip transitions are left
 *      out of the tone estimates.
 *   2. Per class k in {hi, lo}, over its counting samples: n_k, s1_k = sum of x, s2_k = sum of x^2 -- integers, exact
 *      in any order (|x| < 2^26, n <= 781: s2_k < 2^63).  Zero with -a (the cross-product discriminator is not a
 *      frequency).
 *   3. On the host, in double: m_k = s1_k / n_k;
 *        deviation_hz = (m_hi - m_lo) / 2 / 2^24 * 400 kHz / G (G the chain's FIR DC gain, as for offset_hz);
 *        var = (s2_hi - n_hi m_hi^2 + s2_lo - n_lo m_lo^2) / (n_hi + n_lo - 2);
 *        eye_snr_db = 10 log10(((m_hi - m_lo) / 2)^2 / var).
 *      valid = 0 (both NaN) with -a, when a class has fewer than 2 counting samples, when var <= 0, when the report is
 *      off, and for lines of frames handed to wmb_decode_frames.
 *   4. Lines only: chip_rate_hz = 800 kHz (bits - 1) / (end_sample - sync_sample), bits = the bit events the framer
 *      consumed from the access-code bit through the telegram's last bit -- decoded chips per second (T1/C1 chips, S1
 *      Manchester chips).  It does not need the report (NaN when bits < 2), and holds for wmb_decode_frames' lines too.
 * Valid before the first push or right after wmb_reset / wmb_seek (else WMB_E_STATE); on is 0 or 1 (else
 * WMB_E_INVAL).  The setting survives wmb_reset and wmb_seek.  Cost: one more pass over each window already read, and
 * 40 bytes of device-to-host traffic per candidate and per burst. */
typedef struct wmb_line_quality {
    uint64_t sync_sample;     /* as in wmb_line_info                                                         */
    uint64_t end_sample;
    uint32_t n_hi, n_lo;      /* counting samples per class                                                  */
    int64_t  s1_hi, s1_lo;    /* their sum of x                                                              */
    uint64_t s2_hi, s2_lo;    /* their sum of x^2                                                            */
    uint32_t bits;            /* bit events consumed, access-code bit through the last bit                   */
    uint8_t  chain;           /* WMB_CHAIN_*                                                                 */
    uint8_t  algo;            /* WMB_ALGO_*                                                                  */
    uint8_t  crc_ok;
    uint8_t  valid;           /* deviation_hz and eye_snr_db                                                 */
    double   deviation_hz;
    double   eye_snr_db;
    double   chip_rate_hz;
} wmb_line_quality;

typedef struct wmb_burst_quality {
    uint64_t start_sample;    /* as in wmb_burst                                                             */
    uint32_t n_hi, n_lo;
    int64_t  s1_hi, s1_lo;
    uint64_t s2_hi, s2_lo;
    double   deviation_hz;
    double   eye_snr_db;
    uint8_t  chain;
    uint8_t  valid;
    uint8_t  pad[6];
} wmb_burst_quality;

int wmb_set_line_quality(wmb_ctx *c, int on);

/* wmb_take_lines_info that also fills qual[i] for the i-th line taken (info and qual may each be NULL); with either it
 * takes at most rec_cap lines. */
size_t wmb_take_lines_quality(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode,
                              wmb_line_info *info, wmb_line_quality *qual, size_t rec_cap);

/* wmb_take_bursts that also fills qual[i] for out[i] (qual may be NULL: wmb_take_bursts is this call). */
int wmb_take_bursts_quality(wmb_ctx *c, wmb_burst *out, wmb_burst_quality *qual, size_t cap, size_t *n);

/* ---- band survey: a power spectrum of the whole captured band, to find the carriers to decode --------------------
 * Off by default.  wmb_set_spectrum(ctx, N, B) with N bins (256, 512, 1024 or 2048) and B blocks per record (1 .. 2^20)
 * turns it on.  It works on the raw cu8 input, before any mixer, prefilter or decimation, so it does not depend on -s,
 * the prefilter or the chain options, and it runs with no chain enabled.
 *   1. Block b covers global IQ samples [b N, (b + 1) N) (the index wmb_seek sets; pushes, batches and seek positions
 *      are multiples of 2048 IQ samples, so no block straddles them).  A block is counted when it was pushed since the
 *      last wmb_reset / wmb_seek and its first decimated sample floor(b N / d) lies in the line window
 *      (wmb_set_line_window), which lets time chunks split the blocks between them.
 *   2. Per block, every operation a separately rounded fp32 operation:
 *        i = (int)(u - 127.5f) for I (even byte) and Q (odd byte) -- the front end's u - 127 - (u >= 128);
 *        x_re = (float)i_I * hann[n], x_im = (float)i_Q * hann[n], hann[n] = (float)(0.5 - 0.5 cos(2 pi n / N)) (double);
 *        X[k] = sum x[n] e^(-2 pi i k n / N): radix-2 decimation in time on bit-reversed input; at stage s (half
 *          2^(s-1)) butterfly j uses tw[j N / 2^s] = ((float)cos(2 pi k / N), (float)-sin(2 pi k / N)) (double),
 *          t_re = w_re b_re - w_im b_im, t_im = w_re b_im + w_im b_re (each product rounded, then the sum),
 *          a' = a + t, b' = a - t componentwise;
 *        p = re re + im im.
 *   3. Record r covers blocks [r B, (r + 1) B).  Per bin k in frequency order (fftshifted: bin k lies (k - N/2) fs / N
 *      from the capture's centre, fs = 0.8 d MHz) it holds sum[k] = sum of rint(p) (uint64: integer terms, exact in any
 *      order; below 2^55 at N = 2048, B = 2^20) and peak[k] = max p, and blocks = the blocks counted.
 *   4. A record is handed out once a block of a later record has been pushed, or at flush (partial).  Records with no
 *      block counted are not handed out; records come out in record order.
 *   5. Time chunks: a chunk's rows are the sequential run's rows restricted to its blocks.  Adding sum and blocks and
 *      taking the max of peak over rows of the same record gives the sequential rows.
 * Device memory: (batch blocks / B + 2) rows of N bins (12 bytes each) in a ring and in each of 4 result slots (and
 * pinned host memory for the slots). */
typedef struct wmb_spectrum_row {
    uint64_t record;          /* r                                                                             */
    uint64_t start_iq;        /* r B N: the record's first IQ sample (its first counted block may lie later)  */
    uint32_t blocks;          /* blocks counted                                                                */
    uint32_t bins;            /* N                                                                             */
    double   hz_low;          /* frequency of bin 0 relative to the capture's centre: -fs / 2                  */
    double   hz_step;         /* fs / N                                                                        */
} wmb_spectrum_row;

/* bins 0: off (the default); else bins 256, 512, 1024 or 2048 and blocks_per_record 1 .. 2^20, and at most 2^23 bins in
 * a table ((batch blocks / B + 2) N, batch blocks = max_batch_mib MiB / 2N), else WMB_E_INVAL.  Valid before the first
 * push or right after wmb_reset / wmb_seek (else WMB_E_STATE).  The setting survives wmb_reset and wmb_seek. */
int wmb_set_spectrum(wmb_ctx *c, uint32_t bins, uint32_t blocks_per_record);

/* Copy up to cap closed records: rows[i], sum[i * bins ...], peak[i * bins ...] (sum and peak hold cap x bins);
 * *n receives their number.  Records not taken stay queued. */
int wmb_take_spectrum(wmb_ctx *c, wmb_spectrum_row *rows, uint64_t *sum, float *peak, size_t cap, size_t *n);

/* Test hook: the survey's window and twiddle tables for N bins: hann[N], tw[N / 2][2] = (cos, -sin). */
int wmb_debug_spectrum_tables(uint32_t bins, float *hann, float *tw);

/* Convenience for offline captures: push + flush + decode + take_lines in one call.
 * `flush` as in wmb_poll.  Returns bytes written to out or a negative error. */
long wmb_process(wmb_ctx *c, const uint8_t *cu8, size_t nbytes, int flush,
                 char *out, size_t outcap, size_t *n_lines, int timestamp_mode);
long wmb_process_device(wmb_ctx *c, const void *dev_cu8, size_t nbytes, int flush,
                        char *out, size_t outcap, size_t *n_lines, int timestamp_mode);

/* ---- introspection for tests / benchmark -------------------------------------- */

typedef struct wmb_stats {
    uint64_t input_samples;       /* IQ samples consumed                              */
    uint64_t decimated_samples;
    uint64_t batches;
    uint64_t kernel_launches;     /* launches of this library's own kernels           */
    uint64_t lanes_run;           /* bit-sync lanes executed (incl. re-runs)          */
    uint64_t lanes_rerun;         /* lanes whose speculative start state was refuted  */
    uint64_t candidates[2][2];    /* access-code matches  [chain][algo]               */
    uint64_t lines[2][2];         /* datagram lines       [chain][algo]               */
    uint64_t lines_crc_ok[2][2];
    uint64_t h2d_bytes, d2h_bytes;
    double   demod_kernel_ms;     /* CUDA-event time of the demod kernels of the last push (sum over its batches) */
    double   bitsync_kernel_ms;   /* ... of the bit-sync kernels (clock-recovery lanes + bit streams; they overlap the
                                     next batch's demod kernel, so the two sums can exceed the wall time)      */
    double   batch_device_ms;     /* first demod kernel -> last bit-sync kernel of the last push (device clock) */
    uint64_t rl_fallbacks;        /* T1/C1 batches redone with the monolithic run-length lanes */
    double   host_batch_ms;       /* cumulative wall time in the enqueue+verify part of batches */
    double   host_gather_ms;      /* cumulative wall time gathering candidate frames          */
    double   host_decode_ms;      /* cumulative wall time in the host framers                 */
    uint64_t overflow_batches;    /* batches whose bits or candidates did not fit a device table (a run-length lane's
                                     event buffer, a stream's event ring, frame words, datagram pool, access-code
                                     matches, pending candidates) and may have lost lines; the stream goes on.  Takes an input no receiver produces: sized for one access-code
                                     match per 256 decimated samples, sustained over a whole batch                 */
} wmb_stats;

int wmb_get_stats(wmb_ctx *c, wmb_stats *s);

/* Stage taps for parity tests: after a wmb_push* + wmb_poll, copy the per-decimated-
 * sample outputs of the demod kernel for the LAST batch to host arrays
 * (dphi: post-FIR, pre-DC-block discriminator output; rssi: (unsigned)rssi).
 * Returns the number of samples copied or a negative error. */
long wmb_debug_copy_stage(wmb_ctx *c, int chain, float *dphi, uint8_t *rssi, size_t cap);

/* Bit-sync stage taps of the LAST batch, packed: bit i of word w = decimated sample 32 w + i of the batch.
 *   which 0: data bits   -- the slicer's output, behind the DC block with -o  (rtl_wmbus.c:1059, bits.bin tap :1060-1061)
 *   which 1: time2 strobes -- the samples at which the clock lock delivers a bit (rtl_wmbus.c:1092-1111)
 *   which 2: clock signs -- sign of the clock-recovery band-pass (rtl_wmbus.c:1089-1090, clock.bin tap); kept only by a
 *            context created with opts.reserved[1] = 1
 * Returns the number of words copied or a negative error. */
long wmb_debug_copy_bits(wmb_ctx *c, int chain, int which, uint32_t *words, size_t cap_words);

/* The bit events the LAST batch appended to one (chain, algo) bit stream, i.e. the calls of
 * t1_c1_packet_decoder() / s1_packet_decoder() the reference makes (rtl_wmbus.c:773-781, :822-830, rawbits.bin tap
 * :1107-1108): [63:24] decimated sample (40 bits), [23:16] (unsigned)rssi, [2] run-length reset since the previous
 * event, [1] access code matched on this bit, [0] the bit.  Returns the number of events copied. */
long wmb_debug_copy_events(wmb_ctx *c, int chain, int algo, uint64_t *ev, size_t cap);

/* Test hook: the device's exact-arithmetic building blocks (csrc/wmb_exact.cuh) on caller-made operands, host arrays of
 * n floats.  mode 0: atan2f(y, x) as the discriminator uses it (operands zero or in [2^-8, 2^23))   1: general
 * atan2f(y, x) (glibc 2.39 fdlibm restated)   2: IEEE division y / x for such operands   3: IEEE sqrt(y) for y zero or an
 * integer below 2^23   4: the polar discriminator of (I, Q) = (y[i], x[i]) against (y[i-1], x[i-1]) (atan2.h:7-10) */
int wmb_debug_arith(wmb_ctx *c, int mode, const float *y, const float *x, float *out, size_t n);

/* ---- time-chunk sharding of one capture (several contexts / GPUs on one stream) ----
 * The reference has no counterpart: it is one sequential loop (rtl_wmbus.c:1298-1357).  A worker that
 * owns the decimated samples [lo, hi) of a capture (1) seeks its context to a position a warm-up halo
 * before lo, (2) pushes the halo, takes wmb_boundary_state() and compares it with the state its left
 * neighbour took after pushing up to the same sample -- equal bytes mean that every recurrence, shift
 * register and telegram in flight is bit-identical from there on, so the chunk decodes exactly as in
 * the sequential run; a mismatch means the halo was too short (retry with a longer one; position 0 is
 * exact by definition), (3) pushes its chunk and a right halo of one maximum telegram -- and goes on pushing
 * while wmb_pending_before(hi) says that a telegram matched in the chunk is still in flight -- and keeps
 * only the lines whose access-code match lies in [lo, hi). */

/* wmb_reset() plus: the next byte pushed is IQ sample `first_iq_sample` of the capture (mixer and
 * decimation phases, sample indices).  Must be a multiple of 2048 * decimation. */
int wmb_seek(wmb_ctx *c, uint64_t first_iq_sample);

/* Only telegrams whose access-code match falls on a decimated sample in [sync_lo, sync_hi) produce
 * lines (default: all).  The others are still decoded: they keep the decoders busy as in the reference. */
int wmb_set_line_window(wmb_ctx *c, uint64_t sync_lo, uint64_t sync_hi);

/* Number of telegrams in flight -- access-code matches whose decoder is still waiting for bits -- whose match lies on a
 * decimated sample below sync_hi.  A worker pushes its right halo until this is 0 for its chunk's end: the halo of "one
 * maximum telegram" is a statement about samples with edges in them, and a telegram that runs into a gap in the input
 * (dead air: the run-length tracker emits nothing until the next edge, then all the bits at once) ends arbitrarily
 * late.  Gathers what is enqueued first, like wmb_boundary_state().  Negative: error. */
long wmb_pending_before(wmb_ctx *c, uint64_t sync_hi);

/* Everything that couples the samples pushed so far to the output still to come: the carried filter,
 * clock and run-length states, the shift registers, and the bit events of every telegram in flight
 * (absolute sample indices, so two contexts that started at different positions can be compared).
 * Valid after a push of whole batch granules.  Returns the number of bytes written or a negative error. */
long wmb_boundary_state(wmb_ctx *c, uint8_t *buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* WMBUS_B200_H */
