/*
 * wmb_chain.cuh -- per-receiver-chain constants (filter coefficients, access codes,
 * frame limits) and the data layouts shared by the kernels and the host side.
 *
 * Coefficient literals are the reference's filter designs (rtl_wmbus.c:338-341,
 * :353-356, :372, :384); like there they are decimal double literals narrowed to
 * float by the initialiser.
 */
#pragma once
#include <stdint.h>

#define WMB_N_CHAINS 2
#define WMB_N_ALGOS  2

/* ---- geometry of the demod kernel (K1) ---- */
#define K1_THREADS   256       /* threads that convert, filter and demodulate a tile                            */
#define K1_BLOCK     (K1_THREADS + 32)   /* ... plus one warp that only runs the RSSI recurrences, one tile behind */
#define K1_HALO      64        /* decimated samples recomputed left of each tile (the S1 FIR's 45 and the RSSI warm-up's 48,
                                  rounded up so that the tile is whole 32-sample slicer words) */
#define K1_RSSI_WARM 48        /* warm-up steps before each segment (contraction 0.32 per step) */
#define K1_RPT_WIDE   8        /* rows per producer thread on d = 1 and the d = 2 fast path: the block still fits 4 per SM */
#define K1_RPT_NARROW 4        /* ... on every other geometry (the tile of decimation 25 must fit one block)               */
/* tile geometry of a kernel instance: RPT rows per producer thread, TILE + HALO = RPT * K1_THREADS rows, TILE outputs
 * (960 or 1984); the RSSI warp runs one segment of SEG outputs per thread (30 of 32 or 31 of 64) */
template <int RPT> struct K1Geo {
    static constexpr int ROWS = RPT * K1_THREADS;
    static constexpr int TILE = ROWS - K1_HALO;
    static constexpr int SEG = 8 * RPT;
    static_assert(TILE % 32 == 0 && TILE % SEG == 0 && TILE / SEG <= 32, "whole slicer words, one RSSI segment per lane");
};
#define K1_TILE      (K1Geo<K1_RPT_NARROW>::TILE)   /* 960: the tile of the separate box / discriminator phases */
#define K1_BOX_MAX   16

/* ---- bit-sync lanes (K2) ---- */
#define K2_THREADS   64
#define K2_EDGE_EMIT_CAP 8192  /* bits written per run-length edge (see DESIGN.md) */

/* lane-local event word: [31:11] sample offset in lane, [10:3] rssi, [2] reset-before,
 * [1] access code matched, [0] data bit */
#define EV_LOCAL(off, rssi, rst, sync, bit) \
    (((uint32_t)(off) << 11) | ((uint32_t)(rssi) << 3) | ((uint32_t)(rst) << 2) | ((uint32_t)(sync) << 1) | (uint32_t)(bit))
#define K2_MAX_CHUNK (1u << 21)

/* stream (ring) event: [63:24] global decimated sample, [23:16] rssi, [2] reset, [1] sync, [0] bit */
#define EVG_M(e)     ((uint64_t)(e) >> 24)
#define EVG_M_MASK   ((1ull << 40) - 1)
#define EVG_RSSI(e)  ((uint32_t)((e) >> 16) & 0xFFu)
#define EVG_RESET(e) ((uint32_t)((e) >> 2) & 1u)
#define EVG_SYNC(e)  ((uint32_t)((e) >> 1) & 1u)
#define EVG_BIT(e)   ((uint32_t)(e) & 1u)

/* maximum number of bits a framer can consume after (and including) the flagged bit */
#define WMB_MAXBITS_T1C1 (1 + 12 + 290 * 12)
#define WMB_MAXBITS_S1   (1 + 16 + 290 * 16)
#define WMB_MAXBITS      WMB_MAXBITS_S1

/* receiver settings (wmb_set_receiver): clock-lock threshold 1..WMB_LOCK_MAX, default 2 (rtl_wmbus.c:865-866); access-code
 * bit errors up to CH::AC_ERR_MAX, default 0 (:99, :103) */
#define WMB_LOCK_MAX     16

struct ChainT1C1 {
    static constexpr int ID = 0;
    static constexpr int BOX = 8;                 /* rtl_wmbus.c:167 */
    static constexpr int NTAPS = 11;              /* rtl_wmbus.c:371 */
    static constexpr uint32_t CODE = 0x543Du;     /* rtl_wmbus.c:97  */
    static constexpr uint32_t CODE_MASK = 0xFFFFu;
    static constexpr uint32_t AC_ERR_MAX = 3;     /* at 4 the preamble 0x5555 matches too          */
    static constexpr uint32_t RAW_MASK = 0x3Fu;   /* rtl_wmbus.c:733 */
    /* Chebyshev-I band-pass, per section {b1, b2, a1, a2} (rtl_wmbus.c:340-341); literals so that
     * they become instruction immediates */
    static constexpr float B10 = 1.999994649, B20 = 0.9999946492, A10 = -1.387139203, A20 = 0.9921518712;
    static constexpr float B11 = -1.99999482, B21 = 0.9999948196, A11 = -1.403492665, A21 = 0.9845934971;
    static constexpr float B12 = 1.703868036e-07, B22 = -1.000010531, A12 = -1.430055639, A22 = 0.9923856172;
};

struct ChainS1 {
    static constexpr int ID = 1;
    static constexpr int BOX = 16;                /* rtl_wmbus.c:183 */
    static constexpr int NTAPS = 46;              /* rtl_wmbus.c:383 */
    static constexpr uint32_t CODE = 0x547696u;   /* rtl_wmbus.c:101 */
    static constexpr uint32_t CODE_MASK = 0xFFFFFFu;
    static constexpr uint32_t AC_ERR_MAX = 6;
    static constexpr uint32_t RAW_MASK = 0xFu;    /* rtl_wmbus.c:644 */
    /* rtl_wmbus.c:355-356 */
    static constexpr float B10 = 1.999994187, B20 = 0.9999941867, A10 = -1.92151475, A20 = 0.9918135499;
    static constexpr float B11 = -1.999994026, B21 = 0.9999940262, A11 = -1.922481015, A21 = 0.984593497;
    static constexpr float B12 = -1.605750097e-07, B22 = -1.000011787, A12 = -1.937432099, A22 = 0.9927241336;
};

#ifdef WMB_HOSTSIM
#define WMB_CONSTANT static const
#else
#define WMB_CONSTANT __device__ __constant__ const
#endif

WMB_CONSTANT float c_fir_t1c1[11] = {
    -0.00456638213, -0.002571450348, 0.02689425925, 0.1141330398, 0.2264456422, 0.2793297826,
    0.2264456422, 0.1141330398, 0.02689425925, -0.002571450348, -0.00456638213 };

/* the reference's dormant pre-decimation low-pass, 1.6 MS/s, pass band 160 kHz, stop band 200 kHz (rtl_wmbus.c:197-239:
 * lp_fir_butter_1600kHz_160kHz_200kHz_t1_c1 and _s1 hold the same 23 coefficients); SURVEY 8f N4 */
WMB_CONSTANT float c_fir_pre[23] = {
    0.000140535927, 1.102280392e-05, 0.0001309279731, 0.001356012537, 0.00551787474, 0.01499414005, 0.03160167988,
    0.05525973093, 0.08315031015, 0.1099887688, 0.1295143636, 0.1366692652, 0.1295143636, 0.1099887688, 0.08315031015,
    0.05525973093, 0.03160167988, 0.01499414005, 0.00551787474, 0.001356012537, 0.0001309279731, 1.102280392e-05,
    0.000140535927 };
#define K1_PRE_TAPS 23
/* the same taps as fixedpt_rconst() makes them for lp_firfp_ / lp_ppffp_butter_1600kHz_160kHz_200kHz (rtl_wmbus.c:235-256,
 * :297-333; fixedptc.h:104 with FIXEDPT_BITS 32, FIXEDPT_WBITS 24: (int32)(b * 256 + 0.5), the literal read as a double);
 * entry 23 is fixedpt_rconst(0), the polyphase branch's twelfth tap */
#define WMB_FXC(R) ((int32_t)((R) * 256 + 0.5))
WMB_CONSTANT int32_t c_fir_pre_fx[24] = {
    WMB_FXC(0.000140535927), WMB_FXC(1.102280392e-05), WMB_FXC(0.0001309279731), WMB_FXC(0.001356012537), WMB_FXC(0.00551787474),
    WMB_FXC(0.01499414005), WMB_FXC(0.03160167988), WMB_FXC(0.05525973093), WMB_FXC(0.08315031015), WMB_FXC(0.1099887688),
    WMB_FXC(0.1295143636), WMB_FXC(0.1366692652), WMB_FXC(0.1295143636), WMB_FXC(0.1099887688), WMB_FXC(0.08315031015),
    WMB_FXC(0.05525973093), WMB_FXC(0.03160167988), WMB_FXC(0.01499414005), WMB_FXC(0.00551787474), WMB_FXC(0.001356012537),
    WMB_FXC(0.0001309279731), WMB_FXC(1.102280392e-05), WMB_FXC(0.000140535927), WMB_FXC(0) };

WMB_CONSTANT float c_fir_s1[46] = {
    -0.000649081282, -0.0009491938209, -0.001361601657, -0.001910785234, -0.002570133495,
    -0.003251218426, -0.003801634695, -0.004012672882, -0.003636803575, -0.002413585945,
    -0.0001013597693, 0.003488892085, 0.008461671287, 0.01481127545, 0.02240598045,
    0.03098477999, 0.0401679839, 0.04948137286, 0.05839197924, 0.06635211627, 0.07284719662,
    0.07744230649, 0.07982251613, 0.07982251613, 0.07744230649, 0.07284719662, 0.06635211627,
    0.05839197924, 0.04948137286, 0.0401679839, 0.03098477999, 0.02240598045, 0.01481127545,
    0.008461671287, 0.003488892085, -0.0001013597693, -0.002413585945, -0.003636803575,
    -0.004012672882, -0.003801634695, -0.003251218426, -0.002570133495, -0.001910785234,
    -0.001361601657, -0.0009491938209, -0.000649081282 };

/* Chebyshev-I band-pass biquads, {b1, b2, a1, a2} per section (b0 == 1 in every section,
 * and multiplying by 1.0f is exact, so that product is not spelled out). */
WMB_CONSTANT float c_iir_t1c1[12] = {
    1.999994649, 0.9999946492, -1.387139203, 0.9921518712,
    -1.99999482, 0.9999948196, -1.403492665, 0.9845934971,
    1.703868036e-07, -1.000010531, -1.430055639, 0.9923856172 };
WMB_CONSTANT float c_iir_s1[12] = {
    1.999994187, 0.9999941867, -1.92151475, 0.9918135499,
    -1.999994026, 0.9999940262, -1.922481015, 0.984593497,
    -1.605750097e-07, -1.000011787, -1.937432099, 0.9927241336 };
WMB_CONSTANT float c_iir_gain = 1.874981046e-06;

/* Sequential state of a clock-recovery lane (K2a).  Two lanes agree on everything that
 * follows a sample iff these agree, which is what the speculative-start verification compares. */
struct IirState {
    float    dc_x, dc_y;        /* DC block (-o)           rtl_wmbus.c:497-515            */
    float    h[6];              /* biquad memories h1,h2 x 3 sections   iir.h:67-71       */
    uint32_t clk3;              /* last L+1 clock signs (bit0 newest, L the clock-lock threshold, 2 by default; no
                                   other bit set) rtl_wmbus.c:1092                                               */
    uint32_t pad;
};

/* Sequential state of a run-length lane (K2m / K2p) */
struct RlState {
    int32_t  run;               /* run_length                           rtl_wmbus.c:707   */
    int32_t  a;                 /* T1/C1: bit_length   S1: samples_per_bit[0]             */
    int32_t  b;                 /* T1/C1: cum error    S1: samples_per_bit[1]             */
    uint32_t flags;             /* bit0 deglitched level, bit1 reset pending for next event */
    uint32_t raw;               /* raw bit history, masked                                */
    uint32_t sr;                /* run-length shift register, masked                      */
};

#ifdef WMB_HOSTSIM
#define WMB_HDI static inline
#else
#define WMB_HDI static inline __host__ __device__
#endif

WMB_HDI void iir_state_init(IirState &s)
{
    s.dc_x = s.dc_y = 0.f;
    for (int i = 0; i < 6; i++) s.h[i] = 0.f;
    s.clk3 = 0; s.pad = 0;
}

WMB_HDI void rl_state_init(RlState &s, int chain)
{
    s.run = 0;
    s.a = chain == 0 ? 8 * 256 : 24;          /* rtl_wmbus.c:720, :634 */
    s.b = chain == 0 ? 0 : 24;                /* rtl_wmbus.c:721, :635 */
    s.flags = 0; s.raw = 0; s.sr = 0;
}
