/*
 * wmb_kernels.cuh -- the device side of libwmbus_b200 (sm_90a).
 *
 *   K1  demod kernel (one launch per batch, both receiver chains): stages IQ tiles
 *       from HBM into shared memory with bulk async copies (TMA, mbarrier), then
 *       cu8 -> int box filter -> decimate -> polar discriminator (exact fdlibm
 *       atan2f) -> post-demod FIR -> (unsigned)RSSI.  Everything here is exactly
 *       parallel: the only history a sample needs is bounded (box 16 input samples,
 *       discriminator 1, FIR 45, RSSI ~16 decimated samples), so each tile
 *       recomputes a 64-sample halo.           rtl_wmbus.c:1310-1352, :1038-1068
 *   K2  bit sync (wmb_bitsync.cuh): the sequential recurrences run one chunk per
 *       thread ("lane"), each lane first re-running a warm-up stretch from a cold
 *       state; the state it reaches at its chunk start is compared with its
 *       predecessor's end state and refuted lanes are re-run from the exact state, so
 *       the result is exact by induction from the stream start.
 *                                            rtl_wmbus.c:1070-1115, :617-852
 *   K2c prefix-sum + compaction of the per-lane run-length bit events into the
 *       stream ring, collecting access-code matches.
 *   K3  frame gather: for every access-code match, the bits that follow it.
 *
 * The kernels are written as phase functions over an explicit (block, thread) index
 * so that tests/hostsim can execute the identical code on the CPU (test-only).
 */
#pragma once
#include "wmb_exact.cuh"
#include "wmb_chain.cuh"

/* =========================================================================== */
/* K1: demod                                                                   */
/* =========================================================================== */

struct K1Params {
    const uint8_t *in;          /* first byte of this batch's IQ data (16-byte aligned)     */
    const uint8_t *hist;        /* the k1_hist_bytes() bytes that precede `in` in the stream */
    int64_t in_bytes;           /* bytes available at `in`                                    */
    int64_t n_hist_iq;          /* real IQ samples before batch sample 0 (older ones are "zero") */
    int64_t M;                  /* decimated samples to produce                              */
    uint32_t d;                 /* decimation                                                */
    uint32_t chains;            /* bit0: T1/C1, bit1: S1                                     */
    uint32_t accurate;          /* 0 with -a                                                 */
    uint32_t mix;               /* -s (or explicit carriers)                                 */
    uint32_t prefilter;         /* 1..4: one of the dormant pre-decimation low-passes instead of the box filters (d = 2 only; own kernel instance) */
    uint32_t rpt;               /* rows per producer thread: K1_RPT_NARROW or K1_RPT_WIDE (k1_rows_per_thread(); own kernel instances) */
    uint32_t lut_n;             /* mixer table length (fs_kHz/25)                            */
    uint32_t mix_k0;            /* (index of batch sample 0 in the stream) mod lut_n          */
    uint32_t mix_step[WMB_N_CHAINS];  /* table entries per sample = |carrier offset| / 25 kHz, mod lut_n (the reference: 13) */
    uint32_t mix_conj[WMB_N_CHAINS];  /* 0: multiply by the table entry (carrier above the centre: the reference's T1/C1
                                         chain), 1: by its conjugate (below: its S1 chain)         */
    const float *lut_cos, *lut_msin;
    float   *dphi[WMB_N_CHAINS];   /* out: post-FIR discriminator, index 0 = batch sample 0 */
    uint8_t *rssi[WMB_N_CHAINS];   /* out: (unsigned)rssi                                    */
    uint32_t *dbits[WMB_N_CHAINS]; /* out: slicer bits dphi >= 0, word w = samples 32w..32w+31 (null with -o: the DC block
                                      sits between FIR and slicer, and the clock lanes slice) */
    uint32_t *tile_ctr;            /* next tile to hand out (zeroed before the launch)       */
};

/* shared-memory layout of one CTA */
struct K1Smem {
    uint8_t *bytes[2];      /* double-buffered raw IQ tile                      */
    int32_t *v;             /* per input sample: truncated I (low 16), Q (high 16) */
    float   *si, *sq;       /* decimated box-filter outputs, TILE+HALO (narrow tiles only; null in the wide ones) */
    float   *draw;          /* discriminator output, TILE+HALO                   */
    float   *mag;           /* 0.6789 |s|, padded; the buffer the current pass writes (one of mag2[])  */
    float   *mag2[2];       /* two passes are in flight: the RSSI warp works one pass behind           */
    uint64_t *bar;          /* two mbarriers                                     */
    int64_t *pass_tile;     /* [2] tile of the pass whose |s| is in mag2[b] (-1: no more passes)       */
    const WmbAtanTab *atab; /* constants of the discriminator's argument reduction (wmb_exact.cuh); first in the block */
    float   *xq;            /* prefilter mode only: Q as float per input sample (I takes v's place); last in the block */
};
#define K1_ATAB_BYTES 256   /* sizeof(WmbAtanTab) rounded up to the alignment of the IQ buffers */
static_assert(sizeof(WmbAtanTab) <= K1_ATAB_BYTES, "table block");

/* The wide tile where its block still fits four times into an SM's shared memory: d = 1, and the d = 2 fast path (no
 * mixer: one pair-sum word per row).  Its box and discriminator phase is fused (k1_box_disc), so it needs no si / sq. */
static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
uint32_t k1_rows_per_thread(uint32_t d, uint32_t mix, uint32_t prefilter)
{
    return !prefilter && (d == 1u || (d == 2u && !mix)) ? K1_RPT_WIDE : K1_RPT_NARROW;
}

static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
int64_t k1_tile_len(uint32_t rpt) { return (int64_t)rpt * K1_THREADS - K1_HALO; }

static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
int64_t k1_tile_iq(uint32_t d, uint32_t rpt) { return (int64_t)d * rpt * K1_THREADS + K1_BOX_MAX; }

/* bytes of stream history that must precede a batch (left overhang of tile 0) */
static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
int64_t k1_hist_bytes(uint32_t d) { return 2 * ((int64_t)d * K1_HALO + K1_BOX_MAX); }

/* bytes of sm.v: one word per IQ sample, or per pair of them on the wide d = 2 fast path (k1_convert_fast) */
static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
size_t k1_v_bytes(uint32_t d, uint32_t rpt) { return (rpt == K1_RPT_WIDE && d == 2u ? 2 : 4) * (size_t)k1_tile_iq(d, rpt); }

static inline
#ifndef WMB_HOSTSIM
__host__ __device__
#endif
size_t k1_smem_bytes(uint32_t d, uint32_t prefilter = 0, uint32_t rpt = K1_RPT_NARROW)
{
    const size_t nb = (size_t)2 * k1_tile_iq(d, rpt);
    const size_t n = (size_t)rpt * K1_THREADS;
    const size_t nsq = rpt == K1_RPT_NARROW ? 2 * 4 * n : 0;
    return 2 * nb + k1_v_bytes(d, rpt) + nsq + 4 * n + 2 * 4 * (n + n / 32 + 4) + 64 + 16 + 16 + K1_ATAB_BYTES
           + (prefilter ? 4 * (size_t)k1_tile_iq(d, rpt) + 16 : 0);
}

/* largest decimation whose tile fits the 227 KB a block may have (232448 B, 1152 B of them static) */
#define WMB_MAX_DECIMATION 25u
static_assert(2 * 2 * (WMB_MAX_DECIMATION * (K1_TILE + K1_HALO) + K1_BOX_MAX) + 4 * (WMB_MAX_DECIMATION * (K1_TILE + K1_HALO) + K1_BOX_MAX)
              + 3 * 4 * (K1_TILE + K1_HALO) + 2 * 4 * ((K1_TILE + K1_HALO) + (K1_TILE + K1_HALO) / 32 + 4) + 96 + K1_ATAB_BYTES + 1152 <= 232448,
              "K1 tile of the largest decimation must fit a block's shared memory");

WMB_HD void k1_carve(K1Smem &sm, uint8_t *base, uint32_t d, uint32_t prefilter = 0, uint32_t rpt = K1_RPT_NARROW)
{
    const size_t nb = (size_t)2 * k1_tile_iq(d, rpt);
    const size_t n = (size_t)rpt * K1_THREADS;
    size_t off = 0;
    sm.atab = (const WmbAtanTab *)base; off += K1_ATAB_BYTES;
    sm.bytes[0] = base + off; off += nb;
    sm.bytes[1] = base + off; off += nb;
    sm.bar = (uint64_t *)(base + off); off += 16;
    sm.pass_tile = (int64_t *)(base + off); off += 16;
    sm.v = (int32_t *)(base + off); off += k1_v_bytes(d, rpt);
    sm.si = sm.sq = nullptr;
    if (rpt == K1_RPT_NARROW) {
        sm.si = (float *)(base + off); off += 4 * n;
        sm.sq = (float *)(base + off); off += 4 * n;
    }
    sm.draw = (float *)(base + off); off += 4 * n;
    sm.mag2[0] = (float *)(base + off); off += 4 * (n + n / 32 + 4);
    sm.mag2[1] = (float *)(base + off); off += 4 * (n + n / 32 + 4);
    sm.mag = sm.mag2[0];
    off = (off + 15) & ~(size_t)15;
    sm.xq = prefilter ? (float *)(base + off) : nullptr;
}

/* first IQ sample (batch-relative, may be negative) held by tile `t` */
WMB_HD int64_t k1_tile_k0(const K1Params &p, int64_t t)
{
    return (int64_t)p.d * (t * k1_tile_len(p.rpt) - K1_HALO) - K1_BOX_MAX;
}

/* phase A: cu8 -> float-127.5 -> (mix) -> truncate to int   rtl_wmbus.c:1312-1334
 * The truncated I and Q are stored biased (+K1_SAMPLE_BIAS) and packed I | Q << 16, so that the box filter
 * can add whole words: |value| <= 181 behind the mixer (127.5 * sqrt 2), 16 of them stay below 2^16. */
#define K1_SAMPLE_BIAS 256
template <int CHAIN>
WMB_D void k1_convert(const K1Params &p, K1Smem &sm, const uint8_t *raw, int64_t tile, int tid)
{
    const int64_t k0 = k1_tile_k0(p, tile);
    const int n = (int)k1_tile_iq(p.d, p.rpt);
    /* samples before the start of the stream (first tile only) are zero */
    const int64_t first = -p.n_hist_iq - k0;
    const int jmin = first > 0 ? (first < n ? (int)first : n) : 0;
    const uint32_t zero = (uint32_t)K1_SAMPLE_BIAS | ((uint32_t)K1_SAMPLE_BIAS << 16);
    const uint16_t *raw16 = (const uint16_t *)raw;                      /* one IQ sample per 16-bit load */
    if (!p.mix) {
        /* (int)(u - 127.5f) == u - 127 - (u >= 128): no float needed */
        for (int j = tid; j < n; j += K1_THREADS) {
            const uint32_t w = raw16[j];
            const uint32_t ui = w & 0xFFu, uq = w >> 8;
            const uint32_t packed = (ui - 127u - (ui >> 7) + K1_SAMPLE_BIAS) | ((uq - 127u - (uq >> 7) + K1_SAMPLE_BIAS) << 16);
            sm.v[j] = (int32_t)(j >= jmin ? packed : zero);
        }
        return;
    }
    /* shift_freq_plus_minus325, rtl_wmbus.c:997-1031: LUT index (13 k) mod n_max, kept incrementally
     * (the thread's samples are K1_THREADS apart).  The 13 (325 kHz / 25 kHz) and the choice between the entry and
     * its conjugate are per-chain parameters here: any carrier on the 25 kHz grid (SURVEY 8f N3). */
    const uint32_t ln = p.lut_n;
    int64_t km = k0 % (int64_t)ln;
    if (km < 0) km += ln;
    const uint32_t st = p.mix_step[CHAIN];
    const bool cj = p.mix_conj[CHAIN] != 0;
    uint32_t idx = (uint32_t)(((uint64_t)st * (((uint64_t)p.mix_k0 + (uint64_t)km + (uint64_t)tid) % ln)) % ln);
    const uint32_t step = (uint32_t)(((uint64_t)st * K1_THREADS) % ln);
    for (int j = tid; j < n; j += K1_THREADS) {
        uint32_t packed = zero;
        if (j >= jmin) {
            const uint32_t w = raw16[j];
            float xi = wmb_fsub((float)(w & 0xFFu), 127.5f);
            float xq = wmb_fsub((float)(w >> 8), 127.5f);
            const float c = p.lut_cos[idx], z = p.lut_msin[idx];
            const float ix = wmb_fmul(xi, c), qx = wmb_fmul(xq, c);
            const float iz = wmb_fmul(xi, z), qz = wmb_fmul(xq, z);
            if (!cj) { xi = wmb_fsub(ix, qz); xq = wmb_fadd(qx, iz); }      /* :1025-1026 */
            else     { xi = wmb_fadd(ix, qz); xq = wmb_fsub(qx, iz); }      /* :1029-1030 */
            const int vi = (int)xi, vq = (int)xq;                       /* float -> int parameter of mavgi() */
            packed = (uint32_t)(vi + K1_SAMPLE_BIAS) | ((uint32_t)(vq + K1_SAMPLE_BIAS) << 16);
        }
        sm.v[j] = (int32_t)packed;
        idx += step;
        if (idx >= ln) idx -= ln;
    }
}

/* phase B: integer box filter + decimation   moving_average_filter.h:47-54, rtl_wmbus.c:1350 */
template <class CH>
WMB_D void k1_box(const K1Params &p, K1Smem &sm, int tid)
{
    const float inv = 1.0f / (float)CH::BOX;
    for (int r = tid; r < K1_TILE + K1_HALO; r += K1_THREADS) {
        const int jend = (int)p.d * r + (int)p.d - 1 + K1_BOX_MAX;
        uint32_t acc = 0;
#pragma unroll
        for (int b = 0; b < CH::BOX; b++) acc += (uint32_t)sm.v[jend - b];
        const int si = (int)(acc & 0xFFFFu) - CH::BOX * K1_SAMPLE_BIAS;
        const int sq = (int)(acc >> 16) - CH::BOX * K1_SAMPLE_BIAS;
        sm.si[r] = wmb_fmul((float)si, inv);
        sm.sq[r] = wmb_fmul((float)sq, inv);
    }
}

/* ---- fast path for the common geometry: decimation 2, no mixer ------------------------
 * One 32-bit word of input = I0 Q0 I1 Q1 = exactly one decimation step.  The truncation
 * (int)(u8 - 127.5f) equals u8 - 127 - (u8 >= 128), so the per-word I and Q sums are two
 * byte dot products (dp4a) minus the count of bytes with the top bit set.  Partial sums are
 * stored biased (+512) and packed I | Q << 16, so box sums over 4 / 8 words are plain
 * 32-bit adds without carries between the halves. */
#define K1_PAIR_BIAS 512

/* bytes of (a, b) picked by the four selector nibbles of sel (0-3: a, 4-7: b), lowest nibble -> lowest byte */
WMB_D uint32_t wmb_prmt(uint32_t a, uint32_t b, uint32_t sel)
{
#ifdef WMB_HOSTSIM
    const uint64_t ab = (uint64_t)a | ((uint64_t)b << 32);
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((ab >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
#else
    return __byte_perm(a, b, sel);
#endif
}

struct alignas(16) K1Word4 { uint32_t x, y, z, w; };

/* one raw word (I0 Q0 I1 Q1) -> packed biased pair sums (I0+I1 | Q0+Q1 << 16) of the truncated samples:
 * (int)(u - 127.5f) = u - 127 for u < 128 and u - 128 above (rtl_wmbus.c:1312-1313, moving_average_filter.h:47) */
WMB_D uint32_t k1_pair_sums(uint32_t w)
{
    /* truncated sample + 127 = u - (u >> 7), byte by byte: no byte goes below zero, so one 32-bit subtraction does all
     * four; then (I0 | Q0 << 16) + (I1 | Q1 << 16) + the constant is one three-input add */
    const uint32_t t = w - ((w >> 7) & 0x01010101u);
    const uint32_t k = (uint32_t)(K1_PAIR_BIAS - 254) * 0x00010001u;
    return wmb_prmt(t, 0u, 0x4140u) + wmb_prmt(t, 0u, 0x4342u) + k;
}

WMB_D void k1_convert_fast(const K1Params &p, K1Smem &sm, const uint8_t *raw, int64_t tile, int tid)
{
    const int64_t k0 = k1_tile_k0(p, tile);
    const int nw = (int)(k1_tile_iq(p.d, p.rpt) / 2);      /* a multiple of 4 */
    /* words before the start of the stream (first tile only) read as two "zero" samples */
    const int64_t first = (-p.n_hist_iq - k0 + 1) >> 1;          /* smallest j with k0 + 2j >= -n_hist_iq */
    const int jmin = first > 0 ? (first < nw ? (int)first : nw) : 0;
    const uint32_t zero = (uint32_t)K1_PAIR_BIAS | ((uint32_t)K1_PAIR_BIAS << 16);
    const K1Word4 *src = (const K1Word4 *)raw;
    K1Word4 *dst = (K1Word4 *)sm.v;
    for (int g = tid; g < nw / 4; g += K1_THREADS) {           /* four words per step: 128-bit shared accesses */
        const K1Word4 w = src[g];
        K1Word4 o;
        o.x = k1_pair_sums(w.x); o.y = k1_pair_sums(w.y); o.z = k1_pair_sums(w.z); o.w = k1_pair_sums(w.w);
        if (4 * g < jmin) {                                      /* first tile of the stream only */
            if (4 * g + 0 < jmin) o.x = zero;
            if (4 * g + 1 < jmin) o.y = zero;
            if (4 * g + 2 < jmin) o.z = zero;
            if (4 * g + 3 < jmin) o.w = zero;
        }
        dst[g] = o;
    }
}

WMB_HD int k1_pad(int r) { return r + (r >> 5); }

/* phase C: discriminator and |s|   rtl_wmbus.c:1047, :1066 */
WMB_D void k1_disc_mag(const K1Params &p, K1Smem &sm, int tid)
{
    for (int r = tid; r < K1_TILE + K1_HALO; r += K1_THREADS) {
        const float i = sm.si[r], q = sm.sq[r];
        float dr = 0.f;
        if (r > 0) {
            const float ip = sm.si[r - 1], qp = sm.sq[r - 1];
            dr = p.accurate ? wmb_discriminator(i, q, ip, qp, sm.atab) : wmb_discriminator_fast(i, q, ip, qp);
        }
        sm.draw[r] = dr;
        /* the RSSI one-pole needs 0.6789f * |s| (rtl_wmbus.c:480); the product is formed here, in the
         * wide phase, so that the serial recurrence below is one FMUL + one FADD per step */
        sm.mag[k1_pad(r)] = wmb_fmul(0.6789f, wmb_fsqrt(wmb_fadd(wmb_fmul(i, i), wmb_fmul(q, q))));
    }
}

/* ---- optional front end (SURVEY 8f N4): the reference's dormant pre-decimation low-pass ----------------------------
 * rtl_wmbus.c:197-239 keeps a 23-tap FIR for 1.6 MS/s next to the moving averages and never calls it.  With
 * opts.prefilter = 1 it takes the box filters' place (d = 2): convert (and mix) to float, y = sum_j b[j] x[k-j]
 * accumulated from 0 in firf()'s order (fir.h:49-72) at the samples the decimation keeps, then the general atan2f and
 * sqrt -- the filter outputs are not integers, so none of the bounded variants applies.  A kernel instance of its own
 * (template parameter PRE): the default kernels are the same code as without it. */
template <int CHAIN>
WMB_D void k1_convert_float(const K1Params &p, K1Smem &sm, const uint8_t *raw, int64_t tile, int tid)
{
    const int64_t k0 = k1_tile_k0(p, tile);
    const int n = (int)k1_tile_iq(p.d, p.rpt);
    const int64_t first = -p.n_hist_iq - k0;                    /* samples before the start of the stream are zero (the filter's zero history) */
    const int jmin = first > 0 ? (first < n ? (int)first : n) : 0;
    const uint16_t *raw16 = (const uint16_t *)raw;
    float *xi_out = (float *)sm.v, *xq_out = sm.xq;
    const uint32_t ln = p.lut_n;
    int64_t km = k0 % (int64_t)ln;
    if (km < 0) km += ln;
    const uint32_t st = p.mix_step[CHAIN];
    const bool cj = p.mix_conj[CHAIN] != 0;
    uint32_t idx = (uint32_t)(((uint64_t)st * (((uint64_t)p.mix_k0 + (uint64_t)km + (uint64_t)tid) % ln)) % ln);
    const uint32_t step = (uint32_t)(((uint64_t)st * K1_THREADS) % ln);
    for (int j = tid; j < n; j += K1_THREADS) {
        float xi = 0.0f, xq = 0.0f;
        if (j >= jmin) {
            const uint32_t w = raw16[j];
            xi = wmb_fsub((float)(w & 0xFFu), 127.5f);           /* rtl_wmbus.c:1312-1313 */
            xq = wmb_fsub((float)(w >> 8), 127.5f);
            if (p.mix) {                                         /* :997-1031, as in k1_convert */
                const float c = p.lut_cos[idx], z = p.lut_msin[idx];
                const float ix = wmb_fmul(xi, c), qx = wmb_fmul(xq, c);
                const float iz = wmb_fmul(xi, z), qz = wmb_fmul(xq, z);
                if (!cj) { xi = wmb_fsub(ix, qz); xq = wmb_fadd(qx, iz); }
                else     { xi = wmb_fadd(ix, qz); xq = wmb_fsub(qx, iz); }
            }
        }
        xi_out[j] = xi; xq_out[j] = xq;
        idx += step;
        if (idx >= ln) idx -= ln;
    }
}

/* p.prefilter: 1 the 23-tap float FIR through firf(); 2 the float polyphase filter (ppf.h:44-58, rtl_wmbus.c:258-295): the
 * even-phase samples through taps 1, 3, .., 21 and a zero tap, the odd-phase samples through taps 0, 2, .., 22, each
 * branch a firf() accumulated from 0, then (0 + even) + odd -- the kept sample of d = 2 is the filter's phase 1;
 * 3 / 4 the 24.8 fixed-point twins of 1 / 2 (firfp(), ppffp(); fixedptc.h): sample (int64)x << 8, products >> 8, sum / 256 */
WMB_D void k1_prefir(const K1Params &p, K1Smem &sm, int tid)
{
    const float *xi = (const float *)sm.v, *xq = sm.xq;
    const uint32_t mode = p.prefilter;
    for (int r = tid; r < K1_TILE + K1_HALO; r += K1_THREADS) {
        const int jend = (int)p.d * r + (int)p.d - 1 + K1_BOX_MAX;     /* newest input sample of row r (as in k1_box) */
        /* the window of the first three rows of a tile starts left of what the tile holds (22 or 23 samples back, the
         * overhang is 16): those rows are recomputed halo that nothing reads (the FIR, RSSI and discriminator of the
         * tile's own outputs reach back 46 rows at most) */
        float yi = 0.0f, yq = 0.0f;
        if (mode == 1u) {
#pragma unroll
            for (int j = 0; j < K1_PRE_TAPS; j++) {
                const int q = jend - j;
                const float a = q >= 0 ? xi[q] : 0.0f, b = q >= 0 ? xq[q] : 0.0f;
                yi = wmb_fadd(yi, wmb_fmul(c_fir_pre[j], a));
                yq = wmb_fadd(yq, wmb_fmul(c_fir_pre[j], b));
            }
        } else if (mode == 2u) {
            float ei = 0.0f, eq = 0.0f, oi = 0.0f, oq = 0.0f;
#pragma unroll
            for (int j = 0; j < 12; j++) {
                const int q = jend - 1 - 2 * j;
                const float c = j < 11 ? c_fir_pre[2 * j + 1] : 0.0f;
                const float a = q >= 0 ? xi[q] : 0.0f, b = q >= 0 ? xq[q] : 0.0f;
                ei = wmb_fadd(ei, wmb_fmul(c, a));
                eq = wmb_fadd(eq, wmb_fmul(c, b));
            }
#pragma unroll
            for (int j = 0; j < 12; j++) {
                const int q = jend - 2 * j;
                const float a = q >= 0 ? xi[q] : 0.0f, b = q >= 0 ? xq[q] : 0.0f;
                oi = wmb_fadd(oi, wmb_fmul(c_fir_pre[2 * j], a));
                oq = wmb_fadd(oq, wmb_fmul(c_fir_pre[2 * j], b));
            }
            yi = wmb_fadd(wmb_fadd(0.0f, ei), oi);
            yq = wmb_fadd(wmb_fadd(0.0f, eq), oq);
        } else {
            int32_t ai = 0, aq = 0;
            if (mode == 3u) {
#pragma unroll
                for (int j = 0; j < K1_PRE_TAPS; j++) {
                    const int q = jend - j;
                    const int32_t a = q >= 0 ? (int32_t)xi[q] * 256 : 0, b = q >= 0 ? (int32_t)xq[q] * 256 : 0;
                    ai += (int32_t)(((int64_t)c_fir_pre_fx[j] * (int64_t)a) >> 8);
                    aq += (int32_t)(((int64_t)c_fir_pre_fx[j] * (int64_t)b) >> 8);
                }
            } else {
                int32_t ei = 0, eq = 0, oi = 0, oq = 0;
#pragma unroll
                for (int j = 0; j < 12; j++) {
                    const int q = jend - 1 - 2 * j;
                    const int32_t c = c_fir_pre_fx[j < 11 ? 2 * j + 1 : 23];
                    const int32_t a = q >= 0 ? (int32_t)xi[q] * 256 : 0, b = q >= 0 ? (int32_t)xq[q] * 256 : 0;
                    ei += (int32_t)(((int64_t)c * (int64_t)a) >> 8);
                    eq += (int32_t)(((int64_t)c * (int64_t)b) >> 8);
                }
#pragma unroll
                for (int j = 0; j < 12; j++) {
                    const int q = jend - 2 * j;
                    const int32_t a = q >= 0 ? (int32_t)xi[q] * 256 : 0, b = q >= 0 ? (int32_t)xq[q] * 256 : 0;
                    oi += (int32_t)(((int64_t)c_fir_pre_fx[2 * j] * (int64_t)a) >> 8);
                    oq += (int32_t)(((int64_t)c_fir_pre_fx[2 * j] * (int64_t)b) >> 8);
                }
                ai = ei + oi; aq = eq + oq;
            }
            yi = wmb_fmul((float)ai, 0.00390625f);                     /* fixedpt_tofloat: T * (1.0f / 256) */
            yq = wmb_fmul((float)aq, 0.00390625f);
        }
        sm.si[r] = yi; sm.sq[r] = yq;
    }
}

/* discriminator and |s| on arbitrary floats: the general atan2f, IEEE sqrt */
WMB_D void k1_disc_mag_general(const K1Params &p, K1Smem &sm, int tid)
{
    for (int r = tid; r < K1_TILE + K1_HALO; r += K1_THREADS) {
        const float i = sm.si[r], q = sm.sq[r];
        float dr = 0.f;
        if (r > 0) {
            const float ip = sm.si[r - 1], qp = sm.sq[r - 1];
            if (p.accurate) {
                const float dd = -qp;                            /* conjf(s_last), rtl_wmbus.c:517-534 */
                const float re = wmb_fsub(wmb_fmul(i, ip), wmb_fmul(q, dd));
                const float im = wmb_fadd(wmb_fmul(i, dd), wmb_fmul(q, ip));
                dr = wmb_fmul(wmb_atan2f(im, re), wmb_u2f(0x3ea2f983u));
            } else {
                dr = wmb_discriminator_fast(i, q, ip, qp);
            }
        }
        sm.draw[r] = dr;
        sm.mag[k1_pad(r)] = wmb_fmul(0.6789f, wmb_fsqrt(wmb_fadd(wmb_fmul(i, i), wmb_fmul(q, q))));
    }
}

/* phases B + C in one: every thread owns RPT consecutive rows; it reads the words its box windows cover with
 * 128-bit shared loads, slides the (packed I|Q) box sum from row to row and goes straight on to the discriminator
 * and |s| -- the box outputs never touch shared memory.  FAST: the d = 2 fast path, one pair-sum word per row;
 * otherwise DW = d sample words per row (d = 1, 2, 3; other decimations keep the separate phases). */
template <class CH, int DW, bool FAST, int RPT = K1_RPT_NARROW>
WMB_D void k1_box_disc(const K1Params &p, K1Smem &sm, int tid)
{
    constexpr int NWIN = FAST ? CH::BOX / 2 : CH::BOX;    /* words per box window */
    constexpr int START = FAST ? K1_BOX_MAX / 2 - NWIN : K1_BOX_MAX - CH::BOX;
    constexpr int BIASW = FAST ? K1_PAIR_BIAS : K1_SAMPLE_BIAS;
    constexpr int NLOAD = NWIN + RPT * DW;                /* windows of rows r0-1 .. r0+RPT-1 */
    static_assert(NLOAD % 4 == 0 && START % 4 == 0 && RPT % 4 == 0, "box windows are read as 128-bit words");
    const float inv = 1.0f / (float)CH::BOX;
    for (int r0 = RPT * tid; r0 < K1Geo<RPT>::ROWS; r0 += RPT * K1_THREADS) {
        uint32_t w[NLOAD];
        const K1Word4 *src = (const K1Word4 *)(sm.v + DW * r0 + START);   /* first word of row r0-1's window */
#pragma unroll
        for (int q = 0; q < NLOAD / 4; q++) { const K1Word4 v = src[q]; w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
        uint32_t acc = 0;
#pragma unroll
        for (int b = 0; b < NWIN; b++) acc += w[b];
        float si[RPT + 1], sq[RPT + 1];
#pragma unroll
        for (int k = 0; k < RPT + 1; k++) {
            if (k > 0) {
#pragma unroll
                for (int i = 0; i < DW; i++) acc = acc - w[(k - 1) * DW + i] + w[(k - 1) * DW + i + NWIN];   /* both halves stay non-negative */
            }
            /* the box sums themselves, not sum/len: the discriminator only sees the quotient and the signs of
             * s * conj(s_prev), which a common factor len^2 leaves untouched (zeros and their signs included), and
             * sqrt(len^2 x) = len sqrt(x) exactly, so the division by len moves into the constant behind the sqrt */
            /* (float)(half - bias) without a conversion: 2^23 + half as a bit pattern, minus (2^23 + bias), both exact */
            si[k] = wmb_fsub(wmb_u2f((acc & 0xFFFFu) | 0x4B000000u), (float)(8388608 + NWIN * BIASW));
            sq[k] = wmb_fsub(wmb_u2f(wmb_prmt(acc, 0x4B000000u, 0x7632u)), (float)(8388608 + NWIN * BIASW));
        }
        float dr[RPT];
#pragma unroll
        for (int k = 0; k < RPT; k++) {
            const int r = r0 + k;
            dr[k] = 0.f;
            if (r > 0) dr[k] = p.accurate ? wmb_discriminator(si[k + 1], sq[k + 1], si[k], sq[k], sm.atab)
                                          : wmb_discriminator_fast(wmb_fmul(si[k + 1], inv), wmb_fmul(sq[k + 1], inv),
                                                                   wmb_fmul(si[k], inv), wmb_fmul(sq[k], inv));
            /* 0.6789f * sqrt(i^2 + q^2) with i = S_i / len (rtl_wmbus.c:480, :1066): the scaling by the power of two
             * 1 / len commutes with the correctly rounded sqrt and with the product */
            sm.mag[k1_pad(r)] = wmb_fmul(0.6789f * inv, wmb_fsqrt_pos(wmb_fadd(wmb_fmul(si[k + 1], si[k + 1]), wmb_fmul(sq[k + 1], sq[k + 1]))));
        }
#pragma unroll
        for (int q = 0; q < RPT / 4; q++) {
            float4 o; o.x = dr[4 * q]; o.y = dr[4 * q + 1]; o.z = dr[4 * q + 2]; o.w = dr[4 * q + 3];
            *(float4 *)(sm.draw + r0 + 4 * q) = o;
        }
    }
}

/* FIR outputs o .. o + N - 1 of a tile (fir.h:56-67: newest sample first, accumulate from 0) */
template <class CH, int N>
WMB_D void k1_fir_n(const K1Smem &sm, int o, float (&acc)[N])
{
    static_assert(N % 4 == 0, "outputs are read and written as 128-bit words");
    const float *b = (CH::ID == 0) ? c_fir_t1c1 : c_fir_s1;
    if (CH::NTAPS <= 16) {
        /* N consecutive outputs per thread: their taps overlap, so the window is read once with
         * 128-bit shared loads */
        constexpr int BACK = (CH::NTAPS - 1 + 3) / 4 * 4, WIN = BACK + N;
        float w[WIN];
        const float4 *src = (const float4 *)(sm.draw + K1_HALO + o - BACK);
#pragma unroll
        for (int q = 0; q < WIN / 4; q++) { const float4 v = src[q]; w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
#pragma unroll
        for (int k = 0; k < N; k++) {
            float a = 0.0f;
#pragma unroll
            for (int t = 0; t < CH::NTAPS; t++) a = wmb_fadd(a, wmb_fmul(b[t], w[BACK + k - t]));
            acc[k] = a;
        }
    } else {
        /* long filter (S1: 46 taps): the taps walked four at a time over a rolling window of 128-bit shared loads
         * (N / 4 + 12 loads instead of 46 N for the N outputs); every output still accumulates its taps in the
         * order t = 0, 1, 2, ... */
        constexpr int NCHUNK = (CH::NTAPS + 3) / 4;
        static_assert(K1_HALO >= 4 * NCHUNK, "halo shorter than the filter");
        const float4 *src = (const float4 *)(sm.draw + K1_HALO + o);
        float w[4 + N];
#pragma unroll
        for (int q = 0; q < N / 4; q++) { const float4 v = src[q]; w[4 + 4 * q] = v.x; w[5 + 4 * q] = v.y; w[6 + 4 * q] = v.z; w[7 + 4 * q] = v.w; }
#pragma unroll
        for (int k = 0; k < N; k++) acc[k] = 0.0f;
#pragma unroll
        for (int j = 0; j < NCHUNK; j++) {
            const float4 v = src[-(j + 1)];
            w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;          /* w[i] = draw[HALO + o - 4 j - 4 + i] */
#pragma unroll
            for (int tt = 0; tt < 4; tt++) {
                const int tap = 4 * j + tt;
                if (tap < CH::NTAPS) {
#pragma unroll
                    for (int k = 0; k < N; k++) acc[k] = wmb_fadd(acc[k], wmb_fmul(b[tap], w[4 + k - tt]));
                }
            }
#pragma unroll
            for (int i = N - 1; i >= 0; i--) w[4 + i] = w[i];        /* slide by four, newest end first */
        }
    }
}

/* slicer bits of the outputs o .. o + N - 1 at sample m = m0 + o (rtl_wmbus.c:1059; none past the batch's end) */
template <int N>
WMB_D uint32_t k1_slice_n(const float (&acc)[N], int64_t m, int64_t M)
{
    uint32_t bits = 0;
#pragma unroll
    for (int k = 0; k < N; k++) bits |= (m + k < M && acc[k] >= 0.0f ? 1u : 0u) << k;
    return bits;
}

/* phase D: FIR, RPT consecutive outputs per thread (128-bit stores), and -- without the DC block -- the slicer: the
 * 32 / RPT threads of a 32-sample word OR their bits together by shuffles (whole words per tile) */
template <class CH, int RPT = K1_RPT_NARROW>
WMB_D void k1_fir(const K1Params &p, K1Smem &sm, int64_t tile, int tid)
{
    constexpr int TILE = K1Geo<RPT>::TILE, TPW = 32 / RPT;         /* threads per slicer word */
    static_assert(TILE <= RPT * K1_THREADS && TILE % 32 == 0 && 32 % RPT == 0, "one group of outputs per thread, whole words per tile");
    const int64_t m0 = tile * TILE;
    const int o = RPT * tid;
    const int64_t m = m0 + o;
    const bool live = o < TILE && m < p.M;
    float *out = p.dphi[CH::ID];
    uint32_t grp = 0;
    if (live) {
        float acc[RPT];
        k1_fir_n<CH, RPT>(sm, o, acc);
        if (m + RPT - 1 < p.M) {
#pragma unroll
            for (int q = 0; q < RPT / 4; q++) {
                float4 v; v.x = acc[4 * q]; v.y = acc[4 * q + 1]; v.z = acc[4 * q + 2]; v.w = acc[4 * q + 3];
                *(float4 *)(out + m + 4 * q) = v;
            }
        } else {
            for (int k = 0; k < RPT; k++) if (m + k < p.M) out[m + k] = acc[k];
        }
        grp = k1_slice_n<RPT>(acc, m, p.M);
    }
    uint32_t *bits = p.dbits[CH::ID];
    if (!bits) return;
#ifndef WMB_HOSTSIM
    uint32_t word = grp << (RPT * (tid & (TPW - 1)));
#pragma unroll
    for (int s = 1; s < TPW; s <<= 1) word |= __shfl_xor_sync(0xFFFFFFFFu, word, s);
#else
    /* (the CPU build runs the threads one after another, without shuffles: the word's first thread computes the
     * other groups' outputs again, from the same shared window with the same arithmetic) */
    uint32_t word = grp;
    if ((tid & (TPW - 1)) == 0)
        for (int q = 1; q < TPW; q++) {
            if (o + RPT * q >= TILE || m + RPT * q >= p.M) break;
            float acc[RPT];
            k1_fir_n<CH, RPT>(sm, o + RPT * q, acc);
            word |= k1_slice_n<RPT>(acc, m + RPT * q, p.M) << (RPT * q);
        }
#endif
    if ((tid & (TPW - 1)) == 0 && live) bits[m >> 5] = word;
}

/* RSSI one-pole (rtl_wmbus.c:475-484) for one segment of SEG outputs, started K1_RSSI_WARM samples early from r = 0;
 * seg = 0 .. TILE / SEG - 1.  Runs in the block's extra warp while the other threads are already at the tile's FIR and
 * the next tile's front end: the 80- or 112-step chain is nobody's barrier. */
template <class CH, int RPT = K1_RPT_NARROW>
WMB_D void k1_rssi(const K1Params &p, const float *mag, int64_t tile, int seg)
{
    constexpr int TILE = K1Geo<RPT>::TILE, SEG = K1Geo<RPT>::SEG;
    if (seg >= TILE / SEG) return;
    const int64_t m0 = tile * TILE;
    const int o0 = seg * SEG;
    if (m0 + o0 >= p.M) return;
    const int r0 = K1_HALO + o0 - K1_RSSI_WARM;
    float rr = 0.0f;
    const float B = 1.0f - 0.6789f;
#pragma unroll 8
    for (int j = 0; j < K1_RSSI_WARM; j++)
        rr = wmb_fadd(mag[k1_pad(r0 + j)], wmb_fmul(B, rr));
    /* the segment's bytes leave as 128-bit stores */
    uint32_t pk[SEG / 4];
#pragma unroll
    for (int j = 0; j < SEG / 4; j++) pk[j] = 0;
#pragma unroll
    for (int j = 0; j < SEG; j++) {
        rr = wmb_fadd(mag[k1_pad(r0 + K1_RSSI_WARM + j)], wmb_fmul(B, rr));
        pk[j >> 2] |= ((uint32_t)(unsigned)rr & 0xFFu) << (8 * (j & 3));
    }
    uint8_t *dst = p.rssi[CH::ID] + m0 + o0;
    if (m0 + o0 + SEG <= p.M) {
#pragma unroll
        for (int q = 0; q < SEG / 16; q++) {
            K1Word4 v; v.x = pk[4 * q]; v.y = pk[4 * q + 1]; v.z = pk[4 * q + 2]; v.w = pk[4 * q + 3];
            ((K1Word4 *)dst)[q] = v;
        }
    } else {
        for (int j = 0; j < SEG; j++) if (m0 + o0 + j < p.M) dst[j] = (uint8_t)(pk[j >> 2] >> (8 * (j & 3)));
    }
}

/* Which global byte ranges make up the raw tile: [hist part][in part], clamped to what
 * exists.  Offsets are relative to the tile start; all multiples of 16 bytes. */
struct K1Load { const uint8_t *src0; int64_t n0; const uint8_t *src1; int64_t off1, n1; };

WMB_HD K1Load k1_plan_load(const K1Params &p, int64_t tile)
{
    K1Load L;
    const int64_t b0 = 2 * k1_tile_k0(p, tile);             /* byte offset relative to p.in */
    const int64_t nb = 2 * k1_tile_iq(p.d, p.rpt);
    const int64_t hb = k1_hist_bytes(p.d);
    L.src0 = nullptr; L.n0 = 0; L.src1 = nullptr; L.off1 = 0; L.n1 = 0;
    int64_t lo = b0, hi = b0 + nb;
    if (lo < 0) {                                            /* only tile 0 */
        const int64_t n = (hi < 0 ? hi : 0) - lo;            /* bytes taken from hist */
        L.src0 = p.hist + (hb + lo); L.n0 = n;
        lo += n;
    }
    if (hi > p.in_bytes) hi = p.in_bytes & ~(int64_t)15;
    if (hi > lo) { L.src1 = p.in + lo; L.off1 = lo - b0; L.n1 = hi - lo; }
    return L;
}

#ifndef WMB_HOSTSIM
/* ---- TMA (1-D bulk async copy) + mbarrier plumbing ---- */
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

/* (the buffer index never indexes the pointer struct: a dynamically indexed member would push the whole struct into
 * local memory, and every shared-memory access of the kernel would become a generic LD/ST with 64-bit addressing) */
__device__ __forceinline__ void k1_issue_load(const K1Params &p, K1Smem &sm, int buf, int64_t tile)
{
    const K1Load L = k1_plan_load(p, tile);
    uint8_t *dst = buf ? sm.bytes[1] : sm.bytes[0];
    uint64_t *bar = sm.bar + buf;
    mbar_expect_tx(bar, (uint32_t)(L.n0 + L.n1));
    if (L.n0) bulk_g2s(dst, L.src0, (uint32_t)L.n0, bar);
    if (L.n1) bulk_g2s(dst + L.off1, L.src1, (uint32_t)L.n1, bar);
}

/* ---- named barriers of the demod block ------------------------------------------------------------------------
 * 1: the K1_THREADS producer threads among themselves (phase boundaries of a pass)
 * 2, 3 (by pass parity): "|s| of this pass is in shared memory" -- producers arrive, the RSSI warp waits
 * 4, 5 (by pass parity): "the RSSI warp is done with this |s| buffer" -- it arrives, the producers wait before the
 *       pass after next writes the buffer again
 * A pass = one receiver chain of one tile.  The RSSI warp therefore has a whole pass of slack: its 80- or 112-step serial
 * chains are nobody's barrier (round-1 profile: barrier stall 3.2-3.5 per issued instruction, most of it here). */
/* (barrier numbers are immediates: with a register operand ptxas reserves all 16 barriers for the block, which caps
 * the SM at 4 resident blocks) */
template <int ID> __device__ __forceinline__ void k1_bar_sync_i(int count) { asm volatile("bar.sync %0, %1;" :: "n"(ID), "r"(count) : "memory"); }
template <int ID> __device__ __forceinline__ void k1_bar_arrive_i(int count) { asm volatile("bar.arrive %0, %1;" :: "n"(ID), "r"(count) : "memory"); }
__device__ __forceinline__ void k1_bar_sync(int id, int count)
{
    switch (id) { case 1: k1_bar_sync_i<1>(count); break; case 2: k1_bar_sync_i<2>(count); break; case 3: k1_bar_sync_i<3>(count); break;
                  case 4: k1_bar_sync_i<4>(count); break; default: k1_bar_sync_i<5>(count); break; }
}
__device__ __forceinline__ void k1_bar_arrive(int id, int count)
{
    switch (id) { case 2: k1_bar_arrive_i<2>(count); break; case 3: k1_bar_arrive_i<3>(count); break;
                  case 4: k1_bar_arrive_i<4>(count); break; default: k1_bar_arrive_i<5>(count); break; }
}
#define K1_BAR_P 1
#define K1_BAR_READY(pass) (2 + (int)((pass) & 1u))
#define K1_BAR_FREE(pass)  (4 + (int)((pass) & 1u))

template <class CH, bool PRE, int RPT>
__device__ __forceinline__ void k1_chain(const K1Params &p, K1Smem &sm, const uint8_t *raw, int64_t tile,
                                         int tid, bool need_convert, uint32_t pass)
{
    const bool fast = (p.d == 2 && !p.mix);
    if (need_convert) {
        if (PRE) k1_convert_float<CH::ID>(p, sm, raw, tile, tid);
        else if (fast) k1_convert_fast(p, sm, raw, tile, tid); else k1_convert<CH::ID>(p, sm, raw, tile, tid);
        k1_bar_sync(K1_BAR_P, K1_THREADS);
    }
    sm.mag = (pass & 1u) ? sm.mag2[1] : sm.mag2[0];
    if (pass >= 2) k1_bar_sync(K1_BAR_FREE(pass), K1_BLOCK);         /* the RSSI warp has read what pass - 2 left there */
    if constexpr (RPT == K1_RPT_WIDE) {                             /* k1_rows_per_thread(): d = 1, or d = 2 without mixer */
        static_assert(!PRE, "the prefilter front end has narrow tiles");
        if (fast) k1_box_disc<CH, 1, true, RPT>(p, sm, tid); else k1_box_disc<CH, 1, false, RPT>(p, sm, tid);
    }
    else if (PRE) {
        k1_prefir(p, sm, tid);
        k1_bar_sync(K1_BAR_P, K1_THREADS);
        k1_disc_mag_general(p, sm, tid);
    }
    else if (fast) k1_box_disc<CH, 1, true, RPT>(p, sm, tid);
    else if (p.d == 3) k1_box_disc<CH, 3, false, RPT>(p, sm, tid);
    else if (p.d == 2) k1_box_disc<CH, 2, false, RPT>(p, sm, tid);
    else if (p.d == 1) k1_box_disc<CH, 1, false, RPT>(p, sm, tid);
    else {
        k1_box<CH>(p, sm, tid);
        k1_bar_sync(K1_BAR_P, K1_THREADS);
        k1_disc_mag(p, sm, tid);
    }
    if (tid == 0) sm.pass_tile[pass & 1u] = tile;
    k1_bar_arrive(K1_BAR_READY(pass), K1_BLOCK);                      /* hand |s| to the RSSI warp ...            */
    k1_bar_sync(K1_BAR_P, K1_THREADS);                                /* ... and go on with the FIR               */
    k1_fir<CH, RPT>(p, sm, tile, tid);
    k1_bar_sync(K1_BAR_P, K1_THREADS);
}

/* CHAINS (bit 0 T1/C1, bit 1 S1) is a template parameter so that a one-chain run does not carry the other
 * chain's registers: the S1 filter's unrolled taps would cost the T1/C1-only kernel a resident CTA per SM */
template <uint32_t CHAINS, bool PRE, int RPT>
WMB_D void k1_demod_body(const K1Params &p)
{
    extern __shared__ __align__(128) uint8_t k1_smem_raw[];
    K1Smem sm;
    k1_carve(sm, k1_smem_raw, p.d, PRE ? 1u : 0u, RPT);
    const int tid = threadIdx.x;
    const int64_t ntiles = (p.M + K1Geo<RPT>::TILE - 1) / K1Geo<RPT>::TILE;
    if (tid == 0) {
        mbar_init(&sm.bar[0], 1);
        mbar_init(&sm.bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    wmb_atan_tab_fill((WmbAtanTab *)k1_smem_raw, tid);
    __syncthreads();
    constexpr uint32_t NCH = (CHAINS & 1u) + ((CHAINS >> 1) & 1u);       /* passes per tile */

    if (tid >= K1_THREADS) {
        /* ---- the RSSI warp: pass after pass, one behind the producers ---- */
        const int seg = tid - K1_THREADS;
        for (uint32_t pass = 0;; pass++) {
            k1_bar_sync(K1_BAR_READY(pass), K1_BLOCK);
            const int64_t tile = sm.pass_tile[pass & 1u];
            if (tile < 0) break;
            const float *mag = (pass & 1u) ? sm.mag2[1] : sm.mag2[0];
            const bool s1 = (CHAINS == 2u) || (CHAINS == 3u && (pass % NCH) == 1u);
            if (s1) k1_rssi<ChainS1, RPT>(p, mag, tile, seg); else k1_rssi<ChainT1C1, RPT>(p, mag, tile, seg);
            k1_bar_arrive(K1_BAR_FREE(pass), K1_BLOCK);
        }
        return;
    }

    /* ---- producers.  Tiles are handed out by a counter, not by block index: a block that gets on its SM late simply
     * takes fewer tiles.  Thread 0 draws the next tile and starts its bulk copy before the block works on the
     * current one. */
    __shared__ uint32_t s_tile[2];
    if (tid == 0) {
        const uint32_t t0 = atomicAdd(p.tile_ctr, 1u);
        s_tile[0] = t0;
        if ((int64_t)t0 < ntiles) k1_issue_load(p, sm, 0, t0);
    }
    k1_bar_sync(K1_BAR_P, K1_THREADS);
    uint32_t phase = 0;                                       /* bit b: parity to wait for on barrier b */
    uint32_t pass = 0;
    int buf = 0;
    for (;; buf ^= 1) {
        const int64_t tile = s_tile[buf];
        if (tile >= ntiles) break;
        if (tid == 0) {                                       /* prefetch (s_tile[buf ^ 1] was last read before the barriers of the previous tile) */
            const uint32_t nx = atomicAdd(p.tile_ctr, 1u);
            s_tile[buf ^ 1] = nx;
            if ((int64_t)nx < ntiles) k1_issue_load(p, sm, buf ^ 1, nx);
        }
        mbar_wait(sm.bar + buf, (phase >> buf) & 1u);
        phase ^= 1u << buf;
        const uint8_t *raw = buf ? sm.bytes[1] : sm.bytes[0];
        if (CHAINS & 1u) k1_chain<ChainT1C1, PRE, RPT>(p, sm, raw, tile, tid, true, pass++);
        if (CHAINS & 2u) k1_chain<ChainS1, PRE, RPT>(p, sm, raw, tile, tid, p.mix || !(CHAINS & 1u), pass++);
    }
    /* tell the RSSI warp that there is no further pass (its buffer must be free first), then wait until it has read
     * the last two */
    if (pass >= 2) k1_bar_sync(K1_BAR_FREE(pass), K1_BLOCK);
    if (tid == 0) sm.pass_tile[pass & 1u] = -1;
    k1_bar_arrive(K1_BAR_READY(pass), K1_BLOCK);
    if (pass >= 1) k1_bar_sync(K1_BAR_FREE(pass + 1), K1_BLOCK);
}

/* (resident blocks per SM pinned: the narrow T1/C1-only kernel ran at 40 registers before the RSSI warp moved in; the
 * wide tile's shared memory allows four blocks, and so do its registers) */
template <uint32_t CHAINS, int RPT>
__global__ void __launch_bounds__(K1_BLOCK, CHAINS == 1u && RPT == K1_RPT_NARROW ? 5 : 4) k1_demod_kernel(const K1Params p)
{
    k1_demod_body<CHAINS, false, RPT>(p);
}
/* the prefilter front end (opts.prefilter): its own instances, narrow tiles, three resident blocks */
template <uint32_t CHAINS>
__global__ void __launch_bounds__(K1_BLOCK, 3) k1_demod_pre_kernel(const K1Params p) { k1_demod_body<CHAINS, true, K1_RPT_NARROW>(p); }

#endif /* !WMB_HOSTSIM */

#include "wmb_bitsync.cuh"

/* =========================================================================== */
/* K2c: per-stream prefix sum, compaction into the stream ring, candidates     */
/* =========================================================================== */


struct K2cParams {
    const uint32_t *ev;             /* lane-local events [lanes * cap]                     */
    const uint32_t *cnt;            /* [lanes]                                             */
    uint64_t *base;                 /* [lanes] out: ordinal of each lane's first event     */
    uint32_t lanes, cap, C;
    int64_t  m_base;                /* global decimated index of batch sample 0            */
    uint64_t *ring; uint64_t ring_mask;
    StreamDev *sd;
    uint64_t *cand; uint32_t cand_cap;      /* out: ordinals of access-code matches        */
    uint64_t *agg;                  /* [SCAN_THREADS] scan scratch                         */
    const uint8_t *rssi;            /* (unsigned)rssi, index 0 = batch sample 0            */
    const uint32_t *run_if;         /* optional: only if this word is nonzero              */
    const uint32_t *lane_err;       /* [lanes] error bits of each lane's verified run (K2mParams.lane_err) */
    uint32_t *errors;
};

WMB_D void k2c_compact(const K2cParams &p, uint32_t lane, int tid, int nthr)
{
    if (lane >= p.lanes) return;
    if (p.run_if && !*p.run_if) return;
    if (tid == 0 && p.lane_err && p.lane_err[lane]) {
#ifdef WMB_HOSTSIM
        *p.errors |= p.lane_err[lane];
#else
        atomicOr(p.errors, p.lane_err[lane]);
#endif
    }
    const uint32_t n = p.cnt[lane];
    const uint64_t base = p.base[lane];
    const uint32_t *src = p.ev + (size_t)lane * p.cap;
    const uint64_t m_lane = (uint64_t)(p.m_base + (int64_t)lane * p.C);
    for (uint32_t i = tid; i < n; i += nthr) {
        const uint32_t e = src[i];
        const uint64_t m = m_lane + (e >> 11);
        /* the run-length lanes leave the rssi field empty; it is looked up here, where the
         * gather is wide and its latency hides (rtl_wmbus.c:1074: rssi of the edge sample) */
        const uint64_t g = (m << 24) | ((uint64_t)p.rssi[(int64_t)(m - (uint64_t)p.m_base)] << 16) | (e & 7u);
        p.ring[(base + i) & p.ring_mask] = g;
        if (e & 2u) {
#ifdef WMB_HOSTSIM
            const uint32_t slot = p.sd->n_cand++;
#else
            const uint32_t slot = atomicAdd(&p.sd->n_cand, 1u);
#endif
            if (slot < p.cand_cap) p.cand[slot] = base + i;
            else p.sd->cand_overflow = 1;
        }
    }
}

/* =========================================================================== */
/* K3: frame gather -- driven entirely from the device                         */
/* =========================================================================== */
/* After the bit-sync kernels of a batch every (chain, algorithm) stream holds its new access-code matches as an
 * unordered list of ordinals (appended with atomics) next to the candidates the previous batch could not complete.
 * The gather orders them, looks at each candidate's header to see how many bits a framer can ask for, cuts
 * run-length lists at resets, copies the bits, keeps the still incomplete candidates for the next batch and hands
 * the complete list to K4.  Nothing here needs the host: counts live in GatherDev, kernels are grid-stride loops
 * over however many candidates there are, results are appended to a log the host reads once per push. */

#define WMB_N_STREAMS (WMB_N_CHAINS * WMB_N_ALGOS)          /* stream k = chain * WMB_N_ALGOS + algo */

/* Carrier offset of a candidate (DESIGN §8): the sum of rint(dphi * 2^24) over 32 nominal preamble chips that end one
 * access-code length before the match, in decimated samples before it -- T1/C1 (8 samples per chip) [s-384, s-128),
 * S1 (24.414 samples per chip) [s-1367, s-586) -- clipped to the samples pushed since the last reset / seek */
#define WMB_OFS_T1C1_LO 384
#define WMB_OFS_T1C1_HI 128
#define WMB_OFS_S1_LO   1367
#define WMB_OFS_S1_HI   586
#define WMB_OFS_HIST    1536        /* least dphi history prefix (samples): the longest window, in whole 256-sample units */
#define WMB_OFS_SCALE   16777216.f  /* 2^24: exact scaling, integer terms, a sum that does not depend on the order */

struct OfsAcc {                     /* a carried candidate's sum (beside its ordinal in pend[k]) */
    int64_t  sum;
    uint32_t n;
    uint32_t pad;
};

WMB_D int64_t wmb_ofs_x(float d)    /* one term of the offset sum: rint(dphi * 2^24) */
{
#ifdef WMB_HOSTSIM
    return (int64_t)llrintf(d * WMB_OFS_SCALE);
#else
    return __float2ll_rn(d * WMB_OFS_SCALE);            /* 64-bit: -a's cross products reach 2^15 before scaling */
#endif
}

/* Signal quality of an offset window (DESIGN §8, wmb_line_quality): sample q is high iff x[q] n >= sum (the window
 * mean, no division); q in [lo + 1, hi - 1) counts iff q - 1, q, q + 1 share its class.  Per class: the counting
 * samples, their sum and their sum of squares -- integers, exact in any order (|x| < 2^26, n <= 781: s2 < 2^63) */
struct QualAcc {
    uint32_t n_hi, n_lo;
    int64_t  s1_hi, s1_lo;
    uint64_t s2_hi, s2_lo;
};

WMB_HD void qual_zero(QualAcc &a) { a.n_hi = a.n_lo = 0; a.s1_hi = a.s1_lo = 0; a.s2_hi = a.s2_lo = 0; }
WMB_HD void qual_add(QualAcc &a, const QualAcc &b)
{
    a.n_hi += b.n_hi; a.n_lo += b.n_lo; a.s1_hi += b.s1_hi; a.s1_lo += b.s1_lo; a.s2_hi += b.s2_hi; a.s2_lo += b.s2_lo;
}

/* thread t of nt: its share of the class sums over the window [lo, hi) of dphi (its n samples add up to sum).  Reads
 * stay inside [lo, hi).  k3_fill and kb_reduce both take their sums here. */
WMB_D void qual_part(const float *dphi, int64_t lo, int64_t hi, int64_t sum, int64_t n, uint32_t t, uint32_t nt,
                     QualAcc &a)
{
    qual_zero(a);
    for (int64_t q = lo + 1 + (int64_t)t; q < hi - 1; q += nt) {
        const int64_t x0 = wmb_ofs_x(dphi[q - 1]), x = wmb_ofs_x(dphi[q]), x2 = wmb_ofs_x(dphi[q + 1]);
        const bool c0 = x0 * n >= sum, c = x * n >= sum, c2 = x2 * n >= sum;
        if (c0 != c || c2 != c) continue;                 /* a chip transition: the FIR's ramp between the tones */
        const uint64_t sq = (uint64_t)(x * x);
        if (c) { a.n_hi++; a.s1_hi += x; a.s2_hi += sq; }
        else { a.n_lo++; a.s1_lo += x; a.s2_lo += sq; }
    }
}

struct FrameHdr {                   /* one per candidate, device -> host                   */
    uint64_t ordinal;
    uint64_t sync_sample;
    int64_t  ofs_sum;               /* carrier offset: sum of rint(dphi * 2^24) over the window */
    uint32_t nbits;                 /* events shipped (>= 1)                               */
    uint32_t word_off;              /* offset into the frame word buffer                   */
    uint8_t  chain, algo;
    uint8_t  complete;              /* 1: all bits the header can ask for (or cut by a reset) */
    uint8_t  overflow;              /* (unused)                                            */
    uint8_t  cut;                   /* 1: list ends at a run-length reset                  */
    uint8_t  pad;
    uint16_t ofs_n;                 /* samples in the carrier-offset window after clipping  */
};

struct GatherDev {                  /* device-resident state of the gather, one per context */
    uint32_t n;                     /* candidates of the current batch                      */
    uint32_t base;                  /* where they start in the result log (the batch's slot) */
    uint32_t n_words;               /* frame words of the current batch                     */
    uint32_t pool_n;                /* datagram bytes of the current batch (relative to the slot's pool region) */
    uint32_t off[WMB_N_STREAMS + 1];/* this batch: first candidate of every stream          */
    uint32_t n_pend[WMB_N_STREAMS]; /* candidates waiting for more bits                     */
    uint64_t total_prev[WMB_N_STREAMS];   /* stream totals at the previous gather           */
    uint64_t n_cand_total[WMB_N_STREAMS]; /* access-code matches since the context was made (statistics) */
    uint32_t lanes_rerun;           /* statistics: refuted speculative lanes                */
    uint32_t rl_fallbacks;          /* statistics: batches redone with the monolithic run-length lanes */
    uint64_t soft_from[WMB_N_STREAMS];    /* stream totals before the current batch: its events start here (k3_soft) */
};

struct BatchRec {                   /* what the host needs to know about one gathered batch; written last (k3_publish) */
    uint32_t n, n_words, pool_n, errors;
    uint32_t lanes_rerun, rl_fallbacks;
    uint64_t total[WMB_N_STREAMS];
    uint64_t n_cand_total[WMB_N_STREAMS];
};

struct DecHdr;

struct K3Params {
    const uint64_t *ring[WMB_N_STREAMS];
    uint64_t ring_mask[WMB_N_STREAMS];
    StreamDev *sd[WMB_N_STREAMS];   /* null: stream not enabled                             */
    const uint64_t *cand[WMB_N_STREAMS];   /* new matches, unordered                        */
    uint64_t *pend[WMB_N_STREAMS];  /* carried candidates, ordered                          */
    OfsAcc *pend_ofs[WMB_N_STREAMS];/* their carrier-offset sums, same slots                */
    /* line quality (wmb_set_line_quality): null when off -- nothing below reads or writes them then */
    QualAcc *pend_qual[WMB_N_STREAMS];   /* carried candidates' class sums, same slots as pend   */
    QualAcc *qual_log;              /* one per candidate, parallel to hdr_log               */
    uint32_t qual_skip;             /* 1 (-a): the records hold zero sums                   */
    /* soft values (wmb_set_soft_bits): null when off.  soft_ring[k] parallels ring[k] (T1/C1 streams, and the S1 streams
     * when their values are on; null: no values for the stream), soft_words parallels words */
    int16_t *soft_ring[WMB_N_STREAMS];
    int16_t *soft_words;
    uint32_t pend_cap, cand_cap;
    /* the carrier-offset windows of new matches are read from this batch's dphi set: [prefix | batch_m samples], batch
     * sample 0 = decimated sample m_first (40 bits); `clip` samples before it exist since the last reset / seek */
    const float *dphi[WMB_N_CHAINS];
    uint64_t m_first;
    uint32_t prefix, clip, batch_m;
    GatherDev *gd;
    BatchRec *rec;                  /* this batch's record (its result slot)                */
    FrameHdr *hdr_log; DecHdr *dec_log;
    uint32_t log_base, log_cap;     /* the slot's part of the log                           */
    uint32_t *words; uint32_t words_cap;
    uint32_t *cut_n;                /* [cand_cap] scratch: list length before the reset cut */
    uint64_t *agg;                  /* [SCAN_THREADS] scan scratch                          */
    uint32_t *errors;
    uint32_t final;                 /* end of input: nothing is carried over                */
};

#define K3_SOFT_ERRORS (1u | 4u | 8u | 16u | 32u | 64u)
WMB_D void k3_flag(uint32_t *errors, uint32_t bit)
{
#ifdef WMB_HOSTSIM
    *errors |= bit;
#else
    atomicOr(errors, bit);
#endif
}

/* step 1 (one thread): per-stream counts -> offsets, a place in the log, the batch record */
WMB_D void k3_plan(const K3Params &p)
{
    GatherDev &g = *p.gd;
    uint32_t n = 0;
    for (int k = 0; k < WMB_N_STREAMS; k++) {
        g.off[k] = n;
        if (!p.sd[k]) continue;
        StreamDev &sd = *p.sd[k];
        if (sd.cand_overflow) { k3_flag(p.errors, 16u); sd.cand_overflow = 0; sd.n_cand = p.cand_cap; }
        g.n_cand_total[k] += sd.n_cand;
        g.soft_from[k] = g.total_prev[k];
        uint32_t nk = g.n_pend[k] + sd.n_cand;
        /* ring overrun: the batch wrote more events into this stream's ring than it holds (a run-length tracker whose bit
         * length has collapsed, lane after lane): bits of its candidates may be overwritten -- none of THIS stream's
         * candidates is decoded in this batch, pending ones included; the other streams have their own rings */
        if (sd.total - g.total_prev[k] > p.ring_mask[k] + 1 - WMB_MAXBITS - 64) { k3_flag(p.errors, 32u); g.n_pend[k] = 0; nk = 0; }
        g.total_prev[k] = sd.total;
        n += nk;
    }
    g.off[WMB_N_STREAMS] = n;
    if (n > p.cand_cap || n > p.log_cap) { k3_flag(p.errors, 64u); n = 0; for (int k = 0; k <= WMB_N_STREAMS; k++) g.off[k] = 0; }
    g.n = n;
    g.base = p.log_base;
    g.n_words = 0;
    g.pool_n = 0;
}

/* last step of a batch (one thread, after K4): the record the host reads */
WMB_D void k3_publish(const K3Params &p)
{
    GatherDev &g = *p.gd;
    /* k3_carry counts every incomplete candidate but stores only pend_cap of them (and flags 64): the next gather and
     * the host read n_pend entries of the list.  (A frame-word overflow marks every candidate of the batch incomplete.) */
    for (int k = 0; k < WMB_N_STREAMS; k++) if (g.n_pend[k] > p.pend_cap) g.n_pend[k] = p.pend_cap;
    BatchRec r;
    r.n = g.n; r.n_words = g.n_words; r.pool_n = g.pool_n; r.errors = *p.errors;
    /* the capacity overflows (lane event buffer 1, frame words 4, datagram pool 8, matches 16, ring 32, pending candidates 64)
     * cost bits or candidates of this batch, not the stream: the host counts them, the flags start the next batch clean */
    *p.errors &= ~K3_SOFT_ERRORS;
    r.lanes_rerun = g.lanes_rerun; r.rl_fallbacks = g.rl_fallbacks;
    for (int k = 0; k < WMB_N_STREAMS; k++) { r.total[k] = g.total_prev[k]; r.n_cand_total[k] = g.n_cand_total[k]; }
    *p.rec = r;
}

/* step 2 (thread per candidate, any grid): the ordered candidate list of every stream = the candidates carried
 * over from the previous batch plus the new matches, by rank -- ordinals of one stream are distinct, so the number
 * of smaller ones is the position.  Matches are a few thousand per GiB (false ones at 2^-16 per bit plus the
 * telegrams), so the quadratic count is microseconds; the inner loops read one address per warp. */
WMB_D void k3_fill(const K3Params &p, uint32_t i, uint32_t part, uint32_t nparts)
{
    /* part / nparts: the threads that share candidate i (each counts a slice of the keys; the device wrapper adds the
     * slices up with shuffles -- dense traffic has ~20 k candidates per GiB and stream, 4e8 comparisons) */
    const GatherDev &g = *p.gd;
    const bool live = i < g.n;                                   /* (padding threads stay for the shuffles) */
    int k = 0;
    while (live && k + 1 < WMB_N_STREAMS && i >= g.off[k + 1]) k++;
    const uint32_t j = live ? i - g.off[k] : 0u;
    const uint32_t np = live ? g.n_pend[k] : 0u, nn = live ? g.off[k + 1] - g.off[k] - np : 0u;
    const uint64_t key = !live ? 0ull : j < np ? p.pend[k][j] : p.cand[k][j - np];
    uint32_t rank = 0;
    for (uint32_t q = part; q < np; q += nparts) rank += (p.pend[k][q] < key) ? 1u : 0u;
    for (uint32_t q = part; q < nn; q += nparts) rank += (p.cand[k][q] < key) ? 1u : 0u;
    /* a new match: the sum over its carrier-offset window (a carried one brings its sum along).  The match lies in this
     * batch; the window may reach back into the set's history prefix, never past the first sample pushed */
    const bool fresh = live && j >= np;
    const int chain = k / WMB_N_ALGOS;
    int64_t lo = 0, hi = 0;
    if (fresh) {
        const uint64_t s = EVG_M(p.ring[k][key & p.ring_mask[k]]);
        const int64_t rel = (int64_t)((s - p.m_first) & EVG_M_MASK);
        if (rel < (int64_t)p.batch_m) {
            lo = rel - (chain == 0 ? WMB_OFS_T1C1_LO : WMB_OFS_S1_LO);
            hi = rel - (chain == 0 ? WMB_OFS_T1C1_HI : WMB_OFS_S1_HI);
            if (lo < -(int64_t)p.clip) lo = -(int64_t)p.clip;
            if (hi < lo) hi = lo;
        }
    }
    const float *dphi = fresh ? p.dphi[chain] + p.prefix : nullptr;
    int64_t sum = 0;
    for (int64_t q = lo + (int64_t)part; q < hi; q += nparts) sum += wmb_ofs_x(dphi[q]);
#ifndef WMB_HOSTSIM
    for (uint32_t d = nparts >> 1; d > 0; d >>= 1) {
        rank += __shfl_xor_sync(0xFFFFFFFFu, rank, d);
        sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
    }
#endif
    /* line quality: a second pass over the same window, classed against the mean the shuffles just gave every part */
    QualAcc qa;
    qual_zero(qa);
    if (p.qual_log) {
        if (!p.qual_skip) qual_part(dphi, lo, hi, sum, hi - lo, part, nparts, qa);
#ifndef WMB_HOSTSIM
        for (uint32_t d = nparts >> 1; d > 0; d >>= 1) {
            qa.n_hi += __shfl_xor_sync(0xFFFFFFFFu, qa.n_hi, d);
            qa.n_lo += __shfl_xor_sync(0xFFFFFFFFu, qa.n_lo, d);
            qa.s1_hi += __shfl_xor_sync(0xFFFFFFFFu, qa.s1_hi, d);
            qa.s1_lo += __shfl_xor_sync(0xFFFFFFFFu, qa.s1_lo, d);
            qa.s2_hi += __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)qa.s2_hi, d);
            qa.s2_lo += __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)qa.s2_lo, d);
        }
#endif
    }
    if (!live || part != 0) return;
    if (p.qual_log) p.qual_log[g.base + g.off[k] + rank] = fresh ? qa : p.pend_qual[k][j];
    FrameHdr h;
    h.ordinal = key; h.sync_sample = 0; h.nbits = 0; h.word_off = 0; h.complete = 0; h.overflow = 0; h.cut = 0;
    h.pad = 0;
    if (fresh) { h.ofs_sum = sum; h.ofs_n = (uint16_t)(hi - lo); }
    else { const OfsAcc a = p.pend_ofs[k][j]; h.ofs_sum = a.sum; h.ofs_n = (uint16_t)a.n; }
    h.chain = (uint8_t)chain; h.algo = (uint8_t)(k % WMB_N_ALGOS);
    p.hdr_log[g.base + g.off[k] + rank] = h;
}

/* EN 13757-4 3-out-of-6 decode (t1_c1_packet_decoder.h:50-65), 0xFF = invalid */
WMB_HD uint32_t wmb_dec3of6(uint32_t c)
{
    switch (c) {
    case 0x16: return 0; case 0x0D: return 1; case 0x0E: return 2; case 0x0B: return 3;
    case 0x1C: return 4; case 0x19: return 5; case 0x1A: return 6; case 0x13: return 7;
    case 0x2C: return 8; case 0x25: return 9; case 0x26: return 10; case 0x23: return 11;
    case 0x34: return 12; case 0x31: return 13; case 0x32: return 14; case 0x29: return 15;
    default: return 0xFF;
    }
}

/* total telegram length for an L-field, frame format A (t1_c1_packet_decoder.h:68-96) */
WMB_HD uint32_t wmb_tlg_len_a(uint32_t L)
{
    return 1 + L + 2 * (1 + (L > 9 ? (L - 9 + 15) / 16 : 0));
}

/* Upper bound on the number of events (including the flagged one) the host framer can
 * consume for the candidate at ordinal `ord`, looking only at the header bits that are
 * already available.  Returns 0 when not even the header is there yet. */
WMB_D uint32_t k3_bits_needed(const uint64_t *ring, uint64_t mask, uint64_t ord, uint64_t total, int chain)
{
    const uint64_t avail = total - ord;
    if (chain == 0) {
        if (avail < 13) return 0;
        uint32_t w = 0;
        for (int i = 1; i <= 12; i++) w = (w << 1) | EVG_BIT(ring[(ord + i) & mask]);
        const uint32_t hi = wmb_dec3of6(w >> 6), lo = wmb_dec3of6(w & 63u);
        if (hi != 0xFF && lo != 0xFF) return 1 + 12 * wmb_tlg_len_a((hi << 4) | lo);
        if (w != 0x54Cu && w != 0x543u) return 13;
        if (avail < 25) return 0;
        uint32_t t = 0;
        for (int i = 13; i <= 24; i++) t = (t << 1) | EVG_BIT(ring[(ord + i) & mask]);
        if ((t >> 8) != 0xDu) return 17;
        const uint32_t L = t & 0xFFu;
        uint32_t len = (w == 0x543u) ? 1 + L : wmb_tlg_len_a(L);
        if (len < 2) len = 2;
        return 25 + 8 * (len - 1);
    }
    if (avail < 17) return 0;
    uint32_t L = 0;
    for (int i = 0; i < 8; i++) {
        const uint32_t a = EVG_BIT(ring[(ord + 1 + 2 * i) & mask]), b = EVG_BIT(ring[(ord + 2 + 2 * i) & mask]);
        if (a == b) return 3 + 2 * i;                       /* Manchester violation: framer stops on that chip */
        L = (L << 1) | b;                                    /* 01 -> 1, 10 -> 0 */
    }
    return 1 + 16 * wmb_tlg_len_a(L);
}

/* pass 1 (thread per candidate): how many events to ship */
WMB_D void k3_size(const K3Params &p, uint32_t i)
{
    const GatherDev &g = *p.gd;
    if (i >= g.n) return;
    FrameHdr &h = p.hdr_log[g.base + i];
    const int k = h.chain * WMB_N_ALGOS + h.algo;
    const uint64_t *ring = p.ring[k];
    const uint64_t mask = p.ring_mask[k], total = p.sd[k]->total;
    const uint64_t avail = total - h.ordinal;
    uint32_t need = k3_bits_needed(ring, mask, h.ordinal, total, h.chain);
    uint32_t n = (need == 0 || need > avail) ? (uint32_t)avail : need;
    const uint8_t complete = (need != 0 && need <= avail) ? 1 : 0;
    h.nbits = n; h.complete = complete; h.cut = 0; h.overflow = 0;
    p.cut_n[i] = n;
    h.sync_sample = EVG_M(ring[h.ordinal & mask]);
}

/* pass 1b (block per candidate, run-length streams only): the run-length algorithm resets its
 * decoder when it resets itself (rtl_wmbus.c:717-726) -- cut the list at the first event that
 * follows a reset.  Threads stride over the list; the earliest hit wins through an atomic min. */
WMB_D void k3_cut(const K3Params &p, uint32_t i, int tid, int nthr)
{
    const GatherDev &g = *p.gd;
    if (i >= g.n) return;
    FrameHdr &h = p.hdr_log[g.base + i];
    if (h.algo != 0) return;                                  /* time2 never resets */
    const int k = h.chain * WMB_N_ALGOS + h.algo;
    const uint64_t *ring = p.ring[k];
    const uint64_t mask = p.ring_mask[k];
    const uint32_t n = p.cut_n[i];                            /* list length before cutting (k3_size) */
    for (uint32_t j = 1 + tid; j < n; j += nthr) {
        if (EVG_RESET(ring[(h.ordinal + j) & mask])) {
#ifdef WMB_HOSTSIM
            if (j < h.nbits) h.nbits = j;
#else
            atomicMin(&h.nbits, j);
#endif
            break;
        }
    }
}

/* pass 1c (block per candidate, soft values on): the soft value (wmbus_b200_framer.h) of every event of a T1/C1 candidate,
 * and with S1 values on (the S1 streams have soft rings) of an S1 candidate, that this batch produced, i.e. at a ring
 * position >= the stream's total before the batch, into the soft ring beside the event.  A candidate exists in every
 * batch that produces one of its events, so each shipped event gets its value here, with its dphi at hand in the batch's
 * set; overlapping candidates write the same value.  The window ends at or before the event's own sample (T1/C1: D >= 2,
 * S1: D >= 7) and starts at most 8 * 63 + D + 2 (S1: 24 * 31 + D + 8) samples before it, inside the set's history
 * prefix. */
/* One instance per chain (k3_soft_kernel, and k3_soft_s1_kernel when the S1 streams have soft rings): the chain's
 * constants are compile-time, which keeps the T1/C1 instance at its registers. */
static_assert(WMB_SOFT_D_T2 >= 2 && WMB_SOFT_D_RL >= 2 && WMB_SOFT_S1_D_T2 >= 7 && WMB_SOFT_S1_D_RL >= 7,
              "a soft value's window must end at or before its event's sample");
static_assert(8 * 63 + WMB_SOFT_D_RL + 2 <= WMB_OFS_HIST && 24 * 31 + WMB_SOFT_S1_D_RL + 8 <= WMB_OFS_HIST &&
              WMB_SOFT_S1_D_T2 + 8 <= WMB_OFS_HIST, "a soft value's window must lie inside the dphi history");
template <bool S1>
WMB_D void k3_soft(const K3Params &p, uint32_t i, int tid, int nthr)
{
    const GatherDev &g = *p.gd;
    if (i >= g.n || !p.soft_words) return;
    const FrameHdr &h = p.hdr_log[g.base + i];
    const bool s1 = S1;
    const int chain = S1 ? WMB_CHAIN_S1 : WMB_CHAIN_T1C1;
    if (h.chain != chain) return;
    const int k = chain * WMB_N_ALGOS + h.algo;
    if (S1 && !p.soft_ring[k]) return;
    const uint64_t *ring = p.ring[k];
    const uint64_t mask = p.ring_mask[k], total = p.sd[k]->total;
    const bool rla = h.algo == WMB_ALGO_RLA;
    const float *dphi = p.dphi[chain] + p.prefix;
    const uint64_t from = g.soft_from[k] > h.ordinal ? g.soft_from[k] : h.ordinal;
    /* window [c - lo, c + hi), run cap, samples per chip, delays and scale of the chain */
    const uint32_t cap = s1 ? 31 : 63, spc = s1 ? 24 : 8, shift = s1 ? WMB_SOFT_S1_SHIFT : 12;
    const int64_t lo = s1 ? 8 : 2, hi = s1 ? 8 : 3;
    const int64_t d_rl = s1 ? WMB_SOFT_S1_D_RL : WMB_SOFT_D_RL, d_t2 = s1 ? WMB_SOFT_S1_D_T2 : WMB_SOFT_D_T2;
    /* every event k3_size found (the list before a reset cut, and before a frame-word overflow empties it) */
    for (uint64_t o = from + (uint64_t)tid; o < h.ordinal + p.cut_n[i]; o += (uint64_t)nthr) {
        const uint64_t m = EVG_M(ring[o & mask]);
        uint32_t after = 0;                                   /* n - 1 - i: the run's later events at sample m */
        if (rla)
            while (after <= cap && o + 1 + after < total && EVG_M(ring[(o + 1 + after) & mask]) == m) after++;
        const int64_t c = (int64_t)((m - p.m_first) & EVG_M_MASK) - (rla ? d_rl + (int64_t)spc * after : d_t2);
        int16_t v = WMB_SOFT_NONE;
        if (after <= cap && c - lo >= -(int64_t)p.clip) {
            int64_t sum = 0;
            for (int64_t q = c - lo; q < c + hi; q++) sum += wmb_ofs_x(dphi[q]);
            int64_t x = sum >> shift;                         /* floor */
            x = x > 32767 ? 32767 : x < -32767 ? -32767 : x;
            v = (int16_t)x;
        }
        p.soft_ring[k][o & mask] = v;
    }
}

/* pass 2: exclusive scan of nbits -> word offsets (three-phase block scan) */
WMB_D void k3_offsets_a(const K3Params &p, uint32_t t)
{
    const GatherDev &g = *p.gd;
    const uint32_t per = scan_per_thread(g.n);
    const uint32_t i0 = t * per, i1 = (i0 + per < g.n) ? i0 + per : g.n;
    uint64_t acc = 0;
    for (uint32_t i = i0; i < i1 && i0 < g.n; i++) {
        FrameHdr &h = p.hdr_log[g.base + i];
        if (h.nbits < p.cut_n[i]) { h.complete = 1; h.cut = 1; }     /* k3_cut found a reset */
        acc += h.nbits;
    }
    p.agg[t] = acc;
}
WMB_D void k3_offsets_b(const K3Params &p)
{
    GatherDev &g = *p.gd;
    uint64_t acc = 0;
    for (uint32_t t = 0; t < SCAN_THREADS; t++) { const uint64_t c = p.agg[t]; p.agg[t] = acc; acc += c; }
    if (acc > p.words_cap) { k3_flag(p.errors, 4u); acc = 0; }
    g.n_words = (uint32_t)acc;
    for (int k = 0; k < WMB_N_STREAMS; k++) g.n_pend[k] = 0;         /* k3_carry collects the next batch's */
}
WMB_D void k3_offsets_c(const K3Params &p, uint32_t t)
{
    const GatherDev &g = *p.gd;
    const uint32_t per = scan_per_thread(g.n);
    const uint32_t i0 = t * per, i1 = (i0 + per < g.n) ? i0 + per : g.n;
    uint64_t acc = p.agg[t];
    const bool overflow = (g.n_words == 0);
    for (uint32_t i = i0; i < i1 && i0 < g.n; i++) {
        FrameHdr &h = p.hdr_log[g.base + i];
        if (overflow) { h.nbits = 0; h.complete = 0; }
        h.word_off = (uint32_t)acc;
        acc += h.nbits;
    }
}

/* pass 3 (block per candidate): copy events as wmb_bit words */
WMB_D void k3_copy(const K3Params &p, uint32_t i, int tid, int nthr)
{
    const GatherDev &g = *p.gd;
    if (i >= g.n) return;
    const FrameHdr &h = p.hdr_log[g.base + i];
    const int k = h.chain * WMB_N_ALGOS + h.algo;
    const uint64_t *ring = p.ring[k];
    const uint64_t mask = p.ring_mask[k];
    for (uint32_t j = tid; j < h.nbits; j += nthr) {
        const uint64_t e = ring[(h.ordinal + j) & mask];
        /* the ring keeps 40 bits of the sample index (15.9 days at 800 kS/s): differences are taken modulo 2^40.
         * The offset only orders the lines of one batch (end sample); a spacing beyond 2^23 samples inside one
         * candidate (a carrier that keeps the slicer still for > 10 s) is clamped, not an error. */
        uint64_t off = (EVG_M(e) - h.sync_sample) & EVG_M_MASK;
        if (off >= (1u << 23)) off = (1u << 23) - 1;
        p.words[h.word_off + j] = ((uint32_t)off << 9) | (EVG_RSSI(e) << 1) | EVG_BIT(e);
        if (p.soft_words && p.soft_ring[k]) p.soft_words[h.word_off + j] = p.soft_ring[k][(h.ordinal + j) & mask];
    }
}

/* pass 4 (thread per candidate, any grid): candidates that are still waiting for bits go to the next batch (any
 * order: k3_fill ranks them again); the streams' match lists are emptied.  n_pend was zeroed by k3_offsets_b. */
WMB_D void k3_carry(const K3Params &p, uint32_t i)
{
    GatherDev &g = *p.gd;
    if (i < WMB_N_STREAMS && p.sd[i]) p.sd[i]->n_cand = 0;
    if (i >= g.n || p.final) return;
    const FrameHdr &h = p.hdr_log[g.base + i];
    if (h.complete) return;
    const int k = h.chain * WMB_N_ALGOS + h.algo;
#ifdef WMB_HOSTSIM
    const uint32_t slot = g.n_pend[k]++;
#else
    const uint32_t slot = atomicAdd(&g.n_pend[k], 1u);
#endif
    if (slot < p.pend_cap) {
        p.pend[k][slot] = h.ordinal;
        OfsAcc a; a.sum = h.ofs_sum; a.n = h.ofs_n; a.pad = 0;
        p.pend_ofs[k][slot] = a;
        if (p.qual_log) p.pend_qual[k][slot] = p.qual_log[g.base + i];
    }
    else k3_flag(p.errors, 64u);
}


/* =========================================================================== */
/* K4: frame decode (3-out-of-6 / NRZ / Manchester, L-field, RSSI abort, CRCs)  */
/* =========================================================================== */
/* One thread block per gathered candidate.  The reference walks a telegram bit by bit
 * (t1_c1_packet_decoder.h:272-460 and :649-712, s1_packet_decoder.h:132-282) and stops at the
 * first of: an rssi below the capture threshold on any bit but the telegram's last one (:703-710),
 * a Manchester violation, a mode word that is neither a 3-out-of-6 L-field nor a C1 pattern, a
 * wrong C1 trailer, or the end of the bits there are.  Each of these is tied to a bit index, so the
 * block looks for the smallest such index in parallel, then decodes all bytes in parallel, checks
 * one CRC block per thread (:463-536) and writes the CRC-stripped datagram (:551-636) into a byte
 * pool.  (wmb_framer.c is the host twin behind wmb_decode_frames(); tests compare the two.) */
#define K4_THREADS 32
#define K4_CAPTURE_THRESHOLD 5u     /* PACKET_CAPTURE_THRESHOLD, t1_c1_packet_decoder.h:36 */
enum { K4_ABORT = 0, K4_LINE = 1, K4_NEED_MORE = 2, K4_SKIP = 3 };

struct DecHdr {                     /* one per candidate, device -> host                   */
    uint32_t consumed;              /* bits consumed including the flagged one             */
    uint32_t end_off;               /* sample offset (from sync_sample) of the last consumed bit */
    uint32_t serial;
    uint32_t data_off;              /* byte offset of the datagram in the pool             */
    uint16_t len;                   /* datagram bytes after the CRC strip                  */
    uint8_t  status, mode;          /* K4_* ; 0 T1, 1 C1, 2 S1                             */
    uint8_t  crc_ok, ok_3of6, packet_rssi, current_rssi;
};

struct K4Params {
    const FrameHdr *hdr; uint32_t n;    /* gd == null: n candidates at hdr / dec (test hook)                       */
    const uint32_t *words;
    DecHdr *dec;
    uint8_t *pool; uint32_t pool_cap; uint32_t *pool_n;
    uint32_t *errors;
    const GatherDev *gd;                /* else: the current batch's candidates, gd->n of them from gd->base on    */
};

WMB_D uint32_t k4_count(const K4Params &p) { return p.gd ? p.gd->n : p.n; }

struct K4Smem {
    uint8_t pkt[296];
    int stop_idx;
    uint32_t flags;                 /* 1: 3-out-of-6 error, 2: CRC error */
    uint32_t data_off;
};

#ifdef WMB_HOSTSIM
#define K4_SYNC() do { } while (0)
static inline void k4_smin(int *a, int v) { if (v < *a) *a = v; }
static inline void k4_sor(uint32_t *a, uint32_t v) { *a |= v; }
static inline uint32_t k4_gadd(uint32_t *a, uint32_t v) { const uint32_t o = *a; *a += v; return o; }
#else
#define K4_SYNC() __syncthreads()
WMB_D void k4_smin(int *a, int v) { atomicMin(a, v); }
WMB_D void k4_sor(uint32_t *a, uint32_t v) { atomicOr(a, v); }
WMB_D uint32_t k4_gadd(uint32_t *a, uint32_t v) { return atomicAdd(a, v); }
#endif

/* first stop event in bits [lo, hi): returns true and (status, pos) if the decoder stops there */
WMB_D bool k4_scan(const uint32_t *b, uint32_t nbits, uint32_t lo, uint32_t hi, uint32_t exempt, bool manch,
                   K4Smem &sm, int tid, int nthr, uint32_t &status, uint32_t &pos)
{
    const uint32_t he = hi < nbits ? hi : nbits;
    if (tid == 0) sm.stop_idx = 0x7FFFFFFF;
    K4_SYNC();
    int best = 0x7FFFFFFF;
    for (uint32_t i = lo + (uint32_t)tid; i < he; i += (uint32_t)nthr) {
        const uint32_t w = b[i];
        bool bad = WMB_BIT_RSSI(w) < K4_CAPTURE_THRESHOLD && i != exempt;
        if (manch && !(i & 1u)) bad = bad || (WMB_BIT_DATA(w) == WMB_BIT_DATA(b[i - 1]));   /* "01"/"10" only */
        if (bad && (int)i < best) best = (int)i;
    }
    if (best != 0x7FFFFFFF) k4_smin(&sm.stop_idx, best);
    K4_SYNC();
    const int s = sm.stop_idx;
    K4_SYNC();
    if (s != 0x7FFFFFFF) { status = K4_ABORT; pos = (uint32_t)s; return true; }
    if (hi > nbits) { status = K4_NEED_MORE; pos = nbits - 1; return true; }
    return false;
}

WMB_D uint32_t k4_bits(const uint32_t *b, uint32_t first, uint32_t n)     /* MSB first */
{
    uint32_t v = 0;
    for (uint32_t k = 0; k < n; k++) v = (v << 1) | WMB_BIT_DATA(b[first + k]);
    return v;
}

WMB_D uint32_t k4_crc16(const uint8_t *d, uint32_t n)                      /* polynomial 0x3D65, :463-469 */
{
    uint32_t crc = 0;
    for (uint32_t i = 0; i < n; i++) {
        crc ^= (uint32_t)d[i] << 8;
        for (int k = 0; k < 8; k++) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x3D65u) : (crc << 1);
        crc &= 0xFFFFu;
    }
    return ~crc & 0xFFFFu;
}

WMB_D bool k4_block_ok(const uint8_t *q, uint32_t n)                       /* n includes the CRC bytes */
{
    if (n < 2) return false;
    return k4_crc16(q, n - 2) == (((uint32_t)q[n - 2] << 8) | q[n - 1]);
}

WMB_D void k4_decode(const K4Params &p, uint32_t f, int tid, int nthr, K4Smem &sm)
{
    if (f >= k4_count(p)) return;
    const uint32_t lb = p.gd ? p.gd->base : 0u;
    DecHdr *const dec_out = p.dec + lb;
    const FrameHdr h = p.hdr[lb + f];
    const uint32_t *b = p.words + h.word_off;
    const uint32_t nbits = h.nbits;
    DecHdr d;
    d.consumed = 0; d.end_off = 0; d.serial = 0; d.data_off = 0; d.len = 0; d.status = K4_SKIP; d.mode = 0;
    d.crc_ok = 0; d.ok_3of6 = 0; d.packet_rssi = 0; d.current_rssi = 0;
    if (nbits == 0) { if (tid == 0) dec_out[f] = d; return; }

    for (int i = tid; i < 296; i += nthr) sm.pkt[i] = 0;
    if (tid == 0) sm.flags = 0;
    K4_SYNC();

    uint32_t status = K4_LINE, pos = 0, len = 0, mode = 0;
    bool bframe = false;
    /* the flagged bit: the idle handler keeps the state, then the rssi check (:703-710) */
    if (WMB_BIT_RSSI(b[0]) < K4_CAPTURE_THRESHOLD) { status = K4_ABORT; pos = 0; }
    else if (h.chain == WMB_CHAIN_T1C1) {
        if (!k4_scan(b, nbits, 1, 13, 0xFFFFFFFFu, false, sm, tid, nthr, status, pos)) {
            const uint32_t hi6 = k4_bits(b, 1, 6), lo6 = k4_bits(b, 7, 6);
            const uint32_t hi = wmb_dec3of6(hi6), lo = wmb_dec3of6(lo6);
            const uint32_t word = (hi6 << 6) | lo6;
            if (hi != 0xFFu && lo != 0xFFu) {
                /* T1: 3-out-of-6 coded L-field and data (:298-392) */
                const uint32_t L = (hi << 4) | lo;
                len = wmb_tlg_len_a(L);
                const uint32_t P = 1 + 12 * len;
                if (!k4_scan(b, nbits, 13, P, P - 1, false, sm, tid, nthr, status, pos)) {
                    if (tid == 0) sm.pkt[0] = (uint8_t)L;
                    for (uint32_t l = 1 + (uint32_t)tid; l < len; l += (uint32_t)nthr) {
                        const uint32_t hh = wmb_dec3of6(k4_bits(b, 1 + 12 * l, 6)), ll = wmb_dec3of6(k4_bits(b, 7 + 12 * l, 6));
                        if (hh == 0xFFu || ll == 0xFFu) k4_sor(&sm.flags, 1u);
                        sm.pkt[l] = (uint8_t)((hh == 0xFFu ? 0xFFu : hh << 4) | ll);
                    }
                    pos = P - 1; mode = 0;
                }
            } else if (word != 0x54Cu && word != 0x543u) {          /* neither L-field nor C1 mode word (:334-337) */
                status = K4_ABORT; pos = 12;
            } else {
                /* C1: 4-bit trailer, 8-bit L, NRZ bytes (:399-460) */
                bframe = (word == 0x543u);
                if (!k4_scan(b, nbits, 13, 17, 0xFFFFFFFFu, false, sm, tid, nthr, status, pos)) {
                    if (k4_bits(b, 13, 4) != 0xDu) { status = K4_ABORT; pos = 16; }
                    else if (!k4_scan(b, nbits, 17, 25, 0xFFFFFFFFu, false, sm, tid, nthr, status, pos)) {
                        const uint32_t L = k4_bits(b, 17, 8);
                        len = bframe ? 1 + L : wmb_tlg_len_a(L);
                        const uint32_t after = (len > 2 ? len : 2) - 1;       /* the byte loop runs at least once */
                        const uint32_t P = 25 + 8 * after;
                        if (!k4_scan(b, nbits, 25, P, P - 1, false, sm, tid, nthr, status, pos)) {
                            if (tid == 0) sm.pkt[0] = (uint8_t)L;
                            for (uint32_t l = 1 + (uint32_t)tid; l <= after; l += (uint32_t)nthr)
                                sm.pkt[l] = (uint8_t)k4_bits(b, 25 + 8 * (l - 1), 8);
                            pos = P - 1; mode = 1;
                        }
                    }
                }
            }
        }
    } else {
        /* S1: Manchester coded bytes, chips "01" = 1, "10" = 0 (s1_packet_decoder.h:35-37, :152-168) */
        if (!k4_scan(b, nbits, 1, 17, 0xFFFFFFFFu, true, sm, tid, nthr, status, pos)) {
            uint32_t L = 0;
            for (uint32_t k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(b[2 + 2 * k]);
            len = wmb_tlg_len_a(L);
            const uint32_t P = 1 + 16 * len;
            if (!k4_scan(b, nbits, 17, P, P - 1, true, sm, tid, nthr, status, pos)) {
                if (tid == 0) sm.pkt[0] = (uint8_t)L;
                for (uint32_t l = 1 + (uint32_t)tid; l < len; l += (uint32_t)nthr) {
                    uint32_t v = 0;
                    for (uint32_t k = 0; k < 8; k++) v = (v << 1) | WMB_BIT_DATA(b[2 + 16 * l + 2 * k]);
                    sm.pkt[l] = (uint8_t)v;
                }
                pos = P - 1; mode = 2;
            }
        }
    }
    K4_SYNC();

    d.status = (uint8_t)status;
    d.consumed = pos + 1;
    d.end_off = WMB_BIT_OFFSET(b[pos]);
    if (status != K4_LINE) { if (tid == 0) dec_out[f] = d; return; }

    /* block CRCs, one block per thread */
    const uint32_t n = len;
    uint32_t out_len = 0, nblk = 0;
    if (!bframe) {
        /* format A: 12-byte first block, 18-byte blocks after it (:471-506, strip :551-592) */
        if (n < 12) { if (tid == 0) sm.flags |= 2u; }
        else {
            nblk = 1 + (n - 12 + 17) / 18;
            for (uint32_t j = (uint32_t)tid; j < nblk; j += (uint32_t)nthr) {
                const uint32_t off = j ? 12 + 18 * (j - 1) : 0;
                const uint32_t blk = j ? ((n - off >= 18) ? 18 : n - off) : 12;
                if (!k4_block_ok(sm.pkt + off, blk)) k4_sor(&sm.flags, 2u);
            }
            if (sm.pkt[0] != 0) out_len = n - 2 * nblk;
        }
    } else {
        /* format B: CRC over the first 126 bytes, then over the rest (:508-536, strip :595-636) */
        if (n < 12) { if (tid == 0) sm.flags |= 2u; }
        else {
            nblk = (n + 127) / 128;
            for (uint32_t j = (uint32_t)tid; j < nblk; j += (uint32_t)nthr) {
                const uint32_t off = 128 * j;
                const uint32_t blk = (n - off >= 128) ? 128 : n - off;
                if (!k4_block_ok(sm.pkt + off, blk)) k4_sor(&sm.flags, 2u);
            }
            if (sm.pkt[0] >= 2) {
                uint32_t stripped = 0;
                for (uint32_t j = 0; j < nblk; j++) {
                    const uint32_t blk = (n - 128 * j >= 128) ? 128 : n - 128 * j;
                    if (blk < 2) break;                       /* the reference reads out of bounds here */
                    out_len += blk - 2; stripped++;
                }
                nblk = stripped;
            }
        }
    }
    if (tid == 0) {
        const uint32_t room = (out_len + 3u) & ~3u;
        uint32_t off = room ? k4_gadd(p.pool_n, room) : 0;
        if (room && (off > p.pool_cap || room > p.pool_cap - off)) {
#ifdef WMB_HOSTSIM
            *p.errors |= 8u;
#else
            atomicOr(p.errors, 8u);
#endif
            off = 0xFFFFFFFFu;
        }
        sm.data_off = off;
    }
    K4_SYNC();
    const uint32_t flags = sm.flags, data_off = sm.data_off;
    if (data_off != 0xFFFFFFFFu) {
        uint8_t *out = p.pool + data_off;
        for (uint32_t i = (uint32_t)tid; i < out_len; i += (uint32_t)nthr) {
            uint32_t v;
            if (!bframe) v = i < 10 ? sm.pkt[i] : sm.pkt[12 + 18 * ((i - 10) / 16) + (i - 10) % 16];
            else v = i == 0 ? (uint32_t)(uint8_t)(sm.pkt[0] - 2 * nblk) : sm.pkt[i + 2 * (i / 126)];
            out[i] = (uint8_t)v;
        }
    }
    if (tid == 0) {
        d.mode = (uint8_t)mode;
        d.crc_ok = (flags & 2u) ? 0 : 1;
        d.ok_3of6 = (flags & 1u) ? 0 : 1;
        d.packet_rssi = (uint8_t)WMB_BIT_RSSI(b[1]);            /* rssi at the first bit after sync (:295) */
        d.current_rssi = (uint8_t)WMB_BIT_RSSI(b[pos]);
        d.serial = (uint32_t)sm.pkt[4] | ((uint32_t)sm.pkt[5] << 8) | ((uint32_t)sm.pkt[6] << 16) | ((uint32_t)sm.pkt[7] << 24);
        d.len = (uint16_t)out_len;
        d.data_off = data_off;
        if (data_off == 0xFFFFFFFFu) {                             /* no room in the pool: the line is dropped (counted by the host), */
            d.data_off = 0; d.len = 0;                             /* the decoder's verdict on the bits consumed stays                */
            if (d.status == K4_LINE) d.status = K4_ABORT;
        }
        dec_out[f] = d;
    }
}

/* =========================================================================== */
/* K4R: erasure repair of the candidates K4 has decoded (definition in wmbus_b200_framer.h, host twin wmb_frame_repair()
 * in wmb_framer.c).  One warp per candidate.  The lanes decode the bytes and mark the erasures in parallel; then, block
 * by block, each lane checks the CRC of one filling at a time (at most 4^3 = 64), the passes are counted with an atomic
 * and the lowest passing filling is kept.  It reads K4's verdict from the DecHdr table, so K4 itself is unchanged. */
#include "wmb_frame_a.h"

#define K4R_MAX_ERASURES 3
enum { K4R_NONE = 0, K4R_REPAIRED = 1, K4R_AMBIGUOUS = 2, K4R_TOO_MANY = 3, K4R_UNREPAIRABLE = 4, K4R_TRUNCATED = 5 };

struct RepHdr {                     /* one per candidate, parallel to DecHdr, device -> host */
    uint32_t consumed;              /* P: bits of the telegram incl. the flagged one (0: NONE, TRUNCATED) */
    uint32_t end_off;               /* sample offset (from sync_sample) of bit P - 1 (the streaming record's end) */
    uint32_t serial;
    uint32_t data_off;              /* byte offset of the repaired datagram in the pool (0xFFFFFFFF: no room) */
    uint16_t len;                   /* datagram bytes after the CRC strip                  */
    uint8_t  outcome;               /* K4R_*                                               */
    uint8_t  erasures, blocks, had_line, packet_rssi, current_rssi;
};

struct K4RParams {
    const FrameHdr *hdr; const DecHdr *dec; uint32_t n;    /* gd == null: n candidates at hdr / dec / rep (test hook) */
    const uint32_t *words;
    RepHdr *rep;
    uint8_t *pool; uint32_t pool_cap; uint32_t *pool_n;
    uint32_t *errors;
    uint32_t e_max;                 /* 1..3 */
    const GatherDev *gd;            /* else: the current batch's candidates, gd->n of them from gd->base on (as K4) */
};

WMB_D uint32_t k4r_count(const K4RParams &p) { return p.gd ? p.gd->n : p.n; }

struct K4RSmem {
    uint8_t  pkt[296];              /* the received bytes, erased nibbles / bits zero       */
    uint8_t  em[296];               /* erased: T1 0x10 high nibble, 0x01 low nibble; S1 the bits of the erased pairs */
    uint16_t sym[296];              /* T1: the two received 6-bit words, high << 6 | low   */
    uint32_t bad;                   /* 1: rssi < 5 or a T1 word with no filling; 2: a block with too many erasures */
    uint32_t npass;
    int      best;
    uint32_t ne, nf;                /* the current block's erasures and fillings           */
    uint16_t er_byte[K4R_MAX_ERASURES];
    uint8_t  er_shift[K4R_MAX_ERASURES], er_n[K4R_MAX_ERASURES], er_fill[K4R_MAX_ERASURES][4];
    uint32_t data_off;
};

/* the code words at Hamming distance 1 from a 6-bit word, lowest flipped bit first: 2..4 of them for an invalid word of
 * weight 2 or 4, none for weight 0, 1, 5, 6 or an invalid word of weight 3 */
WMB_D uint32_t k4r_fillings(uint32_t w, uint8_t *fill)
{
    uint32_t n = 0;
    for (uint32_t k = 0; k < 6; k++) {
        const uint32_t v = wmb_dec3of6(w ^ (1u << k));
        if (v != 0xFFu) fill[n++] = (uint8_t)v;
    }
    return n;
}

WMB_D void k4r_repair(const K4RParams &p, uint32_t f, int tid, int nthr, K4RSmem &sm)
{
    if (f >= k4r_count(p)) return;
    const uint32_t lb = p.gd ? p.gd->base : 0u;
    RepHdr *const rep_out = p.rep + lb;
    const FrameHdr h = p.hdr[lb + f];
    const DecHdr d = p.dec[lb + f];
    const uint32_t *b = p.words + h.word_off;
    const uint32_t nbits = h.nbits;
    const bool t1 = h.chain == WMB_CHAIN_T1C1;
    RepHdr r;
    r.consumed = 0; r.end_off = 0; r.serial = 0; r.data_off = 0; r.len = 0; r.outcome = K4R_NONE;
    r.erasures = 0; r.blocks = 0; r.had_line = 0; r.packet_rssi = 0; r.current_rssi = 0;

    /* candidates: a line whose CRCs fail, an S1 abort on a Manchester violation after the L-field byte */
    if (nbits == 0 || d.status == K4_SKIP) { if (tid == 0) rep_out[f] = r; return; }
    if (d.status == K4_LINE && !d.crc_ok) {
        r.had_line = 1;
        if (d.mode == 1) {                              /* C1: no erasures; the record ends at the line's last bit */
            r.outcome = K4R_UNREPAIRABLE; r.consumed = d.consumed; r.end_off = d.end_off;
            if (tid == 0) rep_out[f] = r;
            return;
        }
    } else if (d.status == K4_ABORT && !t1) {
        const uint32_t pos = d.consumed - 1;
        if (pos < 18 || (pos & 1u) || WMB_BIT_DATA(b[pos]) != WMB_BIT_DATA(b[pos - 1])) { if (tid == 0) rep_out[f] = r; return; }
    } else { if (tid == 0) rep_out[f] = r; return; }

    uint32_t L = 0;
    if (t1) L = (wmb_dec3of6(k4_bits(b, 1, 6)) << 4) | wmb_dec3of6(k4_bits(b, 7, 6));
    else for (uint32_t k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(b[2 + 2 * k]);
    const uint32_t len = wmb_tlg_len_a(L);
    const uint32_t P = 1 + (t1 ? 12u : 16u) * len;
    if (nbits < P) { r.outcome = K4R_TRUNCATED; if (tid == 0) rep_out[f] = r; return; }
    r.consumed = P;                                      /* every outcome from here on: the record's end is bit P - 1 */
    r.end_off = WMB_BIT_OFFSET(b[P - 1]);
    if (len < 12) { r.outcome = K4R_UNREPAIRABLE; if (tid == 0) rep_out[f] = r; return; }

    if (tid == 0) sm.bad = 0;
    K4_SYNC();
    for (uint32_t i = (uint32_t)tid; i + 1 < P; i += (uint32_t)nthr)
        if (WMB_BIT_RSSI(b[i]) < K4_CAPTURE_THRESHOLD) k4_sor(&sm.bad, 1u);
    for (uint32_t l = (uint32_t)tid; l < len; l += (uint32_t)nthr) {
        uint32_t v = 0, em = 0, sym = 0;
        if (l == 0) v = L;
        else if (t1) {
            const uint32_t hi6 = k4_bits(b, 1 + 12 * l, 6), lo6 = k4_bits(b, 7 + 12 * l, 6);
            const uint32_t hv = wmb_dec3of6(hi6), lv = wmb_dec3of6(lo6);
            uint8_t fill[6];
            if (hv == 0xFFu) { em |= 0x10u; if (!k4r_fillings(hi6, fill)) k4_sor(&sm.bad, 1u); } else v |= hv << 4;
            if (lv == 0xFFu) { em |= 0x01u; if (!k4r_fillings(lo6, fill)) k4_sor(&sm.bad, 1u); } else v |= lv;
            sym = (hi6 << 6) | lo6;
        } else {
            for (uint32_t k = 0; k < 8; k++) {
                const uint32_t a = WMB_BIT_DATA(b[1 + 16 * l + 2 * k]), c = WMB_BIT_DATA(b[2 + 16 * l + 2 * k]);
                if (a == c) em |= 0x80u >> k;
                else v |= c << (7 - k);
            }
        }
        sm.pkt[l] = (uint8_t)v; sm.em[l] = (uint8_t)em; sm.sym[l] = (uint16_t)sym;
    }
    K4_SYNC();
    const uint32_t nblk = wmb_nblk_a(len);
    for (uint32_t j = (uint32_t)tid; j < nblk; j += (uint32_t)nthr) {
        const uint32_t off = wmb_blk_off_a(j), blk = wmb_blk_len_a(len, j);
        uint32_t ne = 0;
        for (uint32_t i = 0; i < blk; i++) ne += (uint32_t)wmb_popc(sm.em[off + i]);
        if (ne > p.e_max) k4_sor(&sm.bad, 2u);
    }
    K4_SYNC();
    const uint32_t bad = sm.bad;
    uint32_t outcome = (bad & 1u) ? K4R_UNREPAIRABLE : (bad & 2u) ? K4R_TOO_MANY : K4R_NONE;

    /* block by block, in frame order: exactly one filling must pass the CRC */
    uint32_t erasures = 0, blocks = 0;
    for (uint32_t j = 0; j < nblk && outcome == K4R_NONE; j++) {
        const uint32_t off = wmb_blk_off_a(j), blk = wmb_blk_len_a(len, j);
        if (tid == 0) {
            uint32_t ne = 0, nf = 1;
            for (uint32_t i = 0; i < blk; i++) {
                const uint32_t l = off + i, em = sm.em[l];
                if (!em) continue;
                if (t1) {
                    for (uint32_t s = 0; s < 2; s++) {
                        const uint32_t shift = s ? 0u : 4u;
                        if (!(em & (1u << shift))) continue;
                        sm.er_byte[ne] = (uint16_t)l; sm.er_shift[ne] = (uint8_t)shift;
                        sm.er_n[ne] = (uint8_t)k4r_fillings(s ? sm.sym[l] & 63u : sm.sym[l] >> 6, sm.er_fill[ne]);
                        nf *= sm.er_n[ne]; ne++;
                    }
                } else {
                    for (uint32_t k = 0; k < 8; k++) {
                        if (!(em & (0x80u >> k))) continue;
                        sm.er_byte[ne] = (uint16_t)l; sm.er_shift[ne] = (uint8_t)(7 - k); sm.er_n[ne] = 2;
                        sm.er_fill[ne][0] = 0; sm.er_fill[ne][1] = 1;
                        nf *= 2; ne++;
                    }
                }
            }
            sm.ne = ne; sm.nf = nf; sm.npass = 0; sm.best = 0x7FFFFFFF;
        }
        K4_SYNC();
        const uint32_t ne = sm.ne, nf = sm.nf;
        for (uint32_t i = (uint32_t)tid; i < nf; i += (uint32_t)nthr) {
            uint8_t q[18];
            for (uint32_t k = 0; k < blk; k++) q[k] = sm.pkt[off + k];
            uint32_t rest = i;                                   /* mixed radix, the block's first erasure lowest */
            for (uint32_t e = 0; e < ne; e++) {
                q[sm.er_byte[e] - off] |= (uint8_t)(sm.er_fill[e][rest % sm.er_n[e]] << sm.er_shift[e]);
                rest /= sm.er_n[e];
            }
            if (k4_block_ok(q, blk)) { k4_gadd(&sm.npass, 1u); k4_smin(&sm.best, (int)i); }
        }
        K4_SYNC();
        const uint32_t npass = sm.npass;
        if (npass != 1) outcome = npass ? K4R_AMBIGUOUS : K4R_UNREPAIRABLE;
        else {
            if (tid == 0) {
                uint32_t rest = (uint32_t)sm.best;
                for (uint32_t e = 0; e < ne; e++) {
                    sm.pkt[sm.er_byte[e]] |= (uint8_t)(sm.er_fill[e][rest % sm.er_n[e]] << sm.er_shift[e]);
                    rest /= sm.er_n[e];
                }
            }
            erasures += ne; blocks += ne ? 1u : 0u;
        }
        K4_SYNC();
    }
    if (outcome == K4R_NONE) outcome = erasures ? K4R_REPAIRED : K4R_UNREPAIRABLE;
    r.outcome = (uint8_t)outcome;
    if (outcome != K4R_REPAIRED) { if (tid == 0) rep_out[f] = r; return; }

    /* the repaired telegram: CRC-stripped datagram (format A, :551-592) into the pool */
    const uint32_t out_len = len - 2 * nblk;
    if (tid == 0) {
        const uint32_t room = (out_len + 3u) & ~3u;
        uint32_t off = k4_gadd(p.pool_n, room);
        if (off > p.pool_cap || room > p.pool_cap - off) {
#ifdef WMB_HOSTSIM
            *p.errors |= 8u;
#else
            atomicOr(p.errors, 8u);
#endif
            off = 0xFFFFFFFFu;
        }
        sm.data_off = off;
    }
    K4_SYNC();
    const uint32_t data_off = sm.data_off;
    if (data_off != 0xFFFFFFFFu)
        for (uint32_t i = (uint32_t)tid; i < out_len; i += (uint32_t)nthr)
            p.pool[data_off + i] = sm.pkt[wmb_strip_src_a(i)];
    if (tid == 0) {
        r.serial = (uint32_t)sm.pkt[4] | ((uint32_t)sm.pkt[5] << 8) | ((uint32_t)sm.pkt[6] << 16) | ((uint32_t)sm.pkt[7] << 24);
        r.data_off = data_off;
        r.len = (uint16_t)(data_off == 0xFFFFFFFFu ? 0 : out_len);
        r.erasures = (uint8_t)erasures; r.blocks = (uint8_t)blocks;
        r.packet_rssi = (uint8_t)WMB_BIT_RSSI(b[1]);
        r.current_rssi = (uint8_t)WMB_BIT_RSSI(b[P - 1]);
        rep_out[f] = r;
    }
}

/* =========================================================================== */
/* K4S: soft repair of C1, T1 and S1 candidates (definitions in wmbus_b200_framer.h, host twins wmb_frame_repair_soft(),
 * wmb_frame_repair_t1_soft() and wmb_frame_repair_s1_soft() in wmb_framer.c).  One warp per candidate, behind K4R: it
 * reads K4's verdict from DecHdr and overwrites K4R's RepHdr of a C1 line with CRC errors (K4R makes those UNREPAIRABLE;
 * k_max), of a T1 line with CRC errors that K4R found TOO_MANY or UNREPAIRABLE (s_max; had_line = 3, bit 1 saying the
 * T1 soft rule decided) and of an S1 candidate that K4R found so (s1_max; had_line bit 2 set, bit 0 kept: S1 pairs are
 * scored on the fly from their two chips, pattern 0 is pure ML as for T1); every other record stays as K4R wrote it.  The lanes reduce n0, n1, S0, S1 (T1: and score every symbol into shared memory);
 * per failing block they pick the K least reliable bits (T1: symbols) by K rounds of warp argmin over a key that orders
 * (has a value, r or delta, index) -- unique, so the choice does not depend on the lanes -- compute the K single-bit CRC
 * syndromes (T1: of the nibble mask ML ^ runner-up at its byte; the CRC is affine: a pattern's syndrome is the received
 * one XOR its members' syndromes) and test patterns lane and lane + 32 (T1: pattern 0, pure ML, too).  The passes are
 * summed and the lowest passing pattern kept, whatever the lanes' order. */
struct K4SParams {
    const FrameHdr *hdr; const DecHdr *dec; uint32_t n;   /* gd == null: n candidates at hdr / dec / rep (test hook) */
    const uint32_t *words;
    const int16_t *soft;            /* parallel to words                                   */
    const uint8_t *soft_ok;         /* test hook: 0 = this frame has no soft values (null: all have) */
    RepHdr *rep;
    uint8_t *pool; uint32_t pool_cap; uint32_t *pool_n;
    uint32_t *errors;
    uint32_t k_max;                 /* C1: 1..WMB_SOFT_K_MAX, 0 = C1 lines are left alone    */
    uint32_t s_max;                 /* T1: 1..WMB_SOFT_K_MAX, 0 = T1 lines are left alone    */
    uint32_t s1_max;                /* S1: 1..WMB_SOFT_K_MAX, 0 = S1 candidates are left alone */
    const GatherDev *gd;
};

WMB_D uint32_t k4s_count(const K4SParams &p) { return p.gd ? p.gd->n : p.n; }

struct K4SSmem {
    uint8_t  pkt[296];
    uint32_t s0;                    /* the current block's syndrome as received           */
    uint32_t sel[WMB_SOFT_K_MAX];   /* its K least reliable bits (T1: symbols)             */
    uint32_t delta[WMB_SOFT_K_MAX]; /* their single-bit (T1: substitution) syndromes       */
    uint32_t data_off;
    /* T1, per symbol 2 l + s of byte l: hard nibble (0xFF invalid), ML << 4 | runner-up, search key */
    uint8_t  hard[2 * 296], mr[2 * 296];
    uint64_t key[2 * 296];
};

/* warp reductions; the CPU build runs a candidate on one simulated lane, which holds the whole result */
WMB_D int64_t k4s_sum(int64_t x)
{
#ifndef WMB_HOSTSIM
    for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, (long long)x, d);
#endif
    return x;
}
WMB_D uint64_t k4s_min(uint64_t x)
{
#ifndef WMB_HOSTSIM
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t y = __shfl_xor_sync(0xFFFFFFFFu, (unsigned long long)x, d);
        x = y < x ? y : x;
    }
#endif
    return x;
}

/* the linear part of the block CRC for one flipped bit: byte q (mask) of a block with nd data bytes, CRC bytes after them */
WMB_HD uint32_t k4s_delta(uint32_t q, uint32_t mask, uint32_t nd)
{
    if (q == nd) return mask << 8;
    if (q == nd + 1) return mask;
    uint32_t crc = mask << 8;
    for (uint32_t u = q; u < nd; u++) {
        for (int k = 0; k < 8; k++) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x3D65u) : (crc << 1);
        crc &= 0xFFFFu;
    }
    return crc;
}

/* two instances: S1 = false repairs C1 and T1 candidates, S1 = true S1 ones.  The S1 branch in one instance with the
 * others took K4S from 64 to 80 registers (sm_90a) and so from 32 to 25 resident blocks per SM; apart, each instance
 * keeps its own count, and the C1 / T1 instance is the code it was */
template <bool S1>
WMB_D void k4s_repair(const K4SParams &p, uint32_t f, int tid, int nthr, K4SSmem &sm)
{
    if (f >= k4s_count(p)) return;
    const uint32_t lb = p.gd ? p.gd->base : 0u;
    const FrameHdr h = p.hdr[lb + f];
    const DecHdr d = p.dec[lb + f];
    const bool s1 = S1;
    if (S1 != (h.chain == WMB_CHAIN_S1)) return;
    if (h.nbits == 0 || (!s1 && (d.status != K4_LINE || d.crc_ok))) return;
    /* C1 lines (k_max), T1 lines (s_max) and S1 candidates (s1_max) whose erasure repair ended in TOO_MANY or
     * UNREPAIRABLE; an S1 one is a line with CRC errors or a violation abort whose list reaches P */
    const bool t1 = !s1 && d.mode == 0;
    if (t1 || s1) {
        if (!(t1 ? p.s_max : p.s1_max)) return;
        const uint32_t prev = p.rep[lb + f].outcome;
        if (prev != K4R_TOO_MANY && prev != K4R_UNREPAIRABLE) return;
    } else if (d.mode != 1 || !p.k_max) return;
    if (p.soft_ok && !p.soft_ok[f]) return;
    const uint32_t *b = p.words + h.word_off;
    const int16_t *sv = p.soft + h.word_off;
    RepHdr r;
    r.consumed = 0; r.end_off = 0; r.serial = 0; r.data_off = 0; r.len = 0; r.outcome = K4R_UNREPAIRABLE;
    /* had_line: bit 1 the T1 soft rule decided, bit 2 the S1 one (bit 0 of an S1 candidate: K4R's, 0 for an abort) */
    r.erasures = 0; r.blocks = 0; r.had_line = t1 ? 3 : s1 ? (uint8_t)(p.rep[lb + f].had_line | 4u) : 1;
    r.packet_rssi = 0; r.current_rssi = 0;
    const bool bframe = !t1 && !s1 && k4_bits(b, 1, 12) == 0x543u;
    uint32_t L = 0;
    if (s1) for (uint32_t k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(b[2 + 2 * k]);
    else L = t1 ? (wmb_dec3of6(k4_bits(b, 1, 6)) << 4) | wmb_dec3of6(k4_bits(b, 7, 6)) : k4_bits(b, 17, 8);
    const uint32_t len = bframe ? 1 + L : wmb_tlg_len_a(L);
    const uint32_t d0 = t1 ? 13 : 17;                   /* the first chip / bit after the L byte */
    const uint32_t P = s1 ? 1 + 16 * len : t1 ? 1 + 12 * len : 17 + 8 * len;
    r.consumed = P;
    r.end_off = WMB_BIT_OFFSET(b[P - 1]);
    /* T1, S1: not a candidate, K4R's record stands */
    if (len < 12) { if (tid == 0 && !t1 && !s1) p.rep[lb + f] = r; return; }
    if (s1) {                                           /* an rssi drop before P - 1 stays an abort */
        int64_t low = 0;
        for (uint32_t j = (uint32_t)tid; j + 1 < P; j += (uint32_t)nthr) low += WMB_BIT_RSSI(b[j]) < K4_CAPTURE_THRESHOLD;
        if (k4s_sum(low)) return;
    }

    int64_t n0 = 0, n1 = 0, s0 = 0, s1s = 0;
    for (uint32_t j = d0 + (uint32_t)tid; j < P && !s1; j += (uint32_t)nthr) {
        const int16_t v = sv[j];
        if (v == WMB_SOFT_NONE) continue;
        if (WMB_BIT_DATA(b[j])) { n1++; s1s += v; } else { n0++; s0 += v; }
    }
    n0 = k4s_sum(n0); n1 = k4s_sum(n1); s0 = k4s_sum(s0); s1s = k4s_sum(s1s);
    const int64_t a = 2 * n0 * n1, t = s1s * n0 + s0 * n1;
    /* S1 pair q: its ML bit and search key (wmb_frame_a.h) */
    auto s1_pair = [&](uint32_t q, uint32_t *ml) -> uint32_t {
        return wmb_s1_pair(sv[1 + 2 * q], sv[2 + 2 * q], WMB_BIT_DATA(b[1 + 2 * q]), WMB_BIT_DATA(b[2 + 2 * q]), q, ml);
    };
    /* C1 search key of bit j: (has a value, r, j) in one integer; |r| < 2^38, j < 2^12 */
    auto key = [&](uint32_t j) -> uint64_t {
        const int16_t v = sv[j];
        if (v == WMB_SOFT_NONE) return j;
        const int64_t sign = WMB_BIT_DATA(b[j]) ? 1 : -1;
        const int64_t rr = a == 0 ? sign * v : sign * ((int64_t)v * a - t);
        return ((uint64_t)(rr + ((int64_t)1 << 40)) << 12) | j;
    };
    if (t1) {
        /* per symbol i = 2 l + s: hard nibble, ML | runner-up, and the search key (all chips have values, delta, i);
         * delta < 2^43, i < 2^10 */
        for (uint32_t i = 2 + (uint32_t)tid; i < 2 * len; i += (uint32_t)nthr) {
            int64_t y[6];
            uint64_t has = 1;
            for (uint32_t c = 0; c < 6; c++) {
                const int16_t v = sv[1 + 6 * i + c];
                if (v == WMB_SOFT_NONE) has = 0;
                y[c] = v == WMB_SOFT_NONE ? 0 : a == 0 ? (int64_t)v : (int64_t)v * a - t;
            }
            uint32_t ml, ru;
            int64_t delta;
            wmb_t1_sym_ml(y, &ml, &ru, &delta);
            sm.hard[i] = (uint8_t)wmb_dec3of6(k4_bits(b, 1 + 6 * i, 6));
            sm.mr[i] = (uint8_t)(ml << 4 | ru);
            sm.key[i] = has << 53 | (uint64_t)delta << 10 | i;
        }
        for (uint32_t l = (uint32_t)tid; l < len; l += (uint32_t)nthr)
            sm.pkt[l] = l == 0 ? (uint8_t)L
                               : (uint8_t)((wmb_dec3of6(k4_bits(b, 1 + 12 * l, 6)) & 15u) << 4 | (wmb_dec3of6(k4_bits(b, 7 + 12 * l, 6)) & 15u));
    } else if (s1) {                                    /* the hard decode, a violation's bit 0 */
        for (uint32_t l = (uint32_t)tid; l < len; l += (uint32_t)nthr) {
            uint32_t v = L;
            if (l) {
                v = 0;
                for (uint32_t k = 0; k < 8; k++) {
                    const uint32_t x = WMB_BIT_DATA(b[1 + 16 * l + 2 * k]), c = WMB_BIT_DATA(b[2 + 16 * l + 2 * k]);
                    v |= (x != c ? c : 0u) << (7 - k);
                }
            }
            sm.pkt[l] = (uint8_t)v;
        }
    } else
        for (uint32_t l = (uint32_t)tid; l < len; l += (uint32_t)nthr) sm.pkt[l] = (uint8_t)k4_bits(b, 17 + 8 * l, 8);
    K4_SYNC();

    const uint32_t nblk = bframe ? wmb_nblk_b(len) : wmb_nblk_a(len);
    const uint32_t kk = t1 ? p.s_max : s1 ? p.s1_max : p.k_max;
    uint32_t outcome = K4R_NONE, flips = 0, blocks = 0;
    for (uint32_t k = 0; k < nblk && outcome == K4R_NONE; k++) {
        const uint32_t off = bframe ? wmb_blk_off_b(k) : wmb_blk_off_a(k), blk = bframe ? wmb_blk_len_b(len, k) : wmb_blk_len_a(len, k);
        if (blk < 2) { outcome = K4R_UNREPAIRABLE; break; }          /* no CRC: no pattern can pass */
        /* the searchable bits (C1), symbols (T1) or pairs (S1) of the block */
        const uint32_t g0 = off ? off : 1;
        const uint32_t lo = t1 ? 2 * g0 : s1 ? 8 * g0 : 17 + 8 * g0, hi = t1 ? 2 * (off + blk) : s1 ? 8 * (off + blk) : 17 + 8 * (off + blk);
        int64_t invalid = 0;
        if (t1)
            for (uint32_t i = lo + (uint32_t)tid; i < hi; i += (uint32_t)nthr) invalid += sm.hard[i] == 0xFFu;
        else if (s1)
            for (uint32_t q = lo + (uint32_t)tid; q < hi; q += (uint32_t)nthr)
                invalid += WMB_BIT_DATA(b[1 + 2 * q]) == WMB_BIT_DATA(b[2 + 2 * q]);
        invalid = k4s_sum(invalid);
        if (tid == 0) sm.s0 = k4_crc16(sm.pkt + off, blk - 2) ^ (((uint32_t)sm.pkt[off + blk - 2] << 8) | sm.pkt[off + blk - 1]);
        K4_SYNC();
        uint32_t syn = sm.s0;
        K4_SYNC();
        if (syn == 0 && invalid == 0) continue;
        if (t1 || s1) {                                         /* every searchable symbol / pair takes its ML value */
            if (t1)
                for (uint32_t l = lo / 2 + (uint32_t)tid; l < hi / 2; l += (uint32_t)nthr)
                    sm.pkt[l] = (uint8_t)((sm.mr[2 * l] & 0xF0u) | sm.mr[2 * l + 1] >> 4);
            else
                for (uint32_t l = lo / 8 + (uint32_t)tid; l < hi / 8; l += (uint32_t)nthr) {
                    uint32_t v = 0, ml;
                    for (uint32_t k = 0; k < 8; k++) { s1_pair(8 * l + k, &ml); v |= ml << (7 - k); }
                    sm.pkt[l] = (uint8_t)v;
                }
            K4_SYNC();
            if (tid == 0) sm.s0 = k4_crc16(sm.pkt + off, blk - 2) ^ (((uint32_t)sm.pkt[off + blk - 2] << 8) | sm.pkt[off + blk - 1]);
            K4_SYNC();
            syn = sm.s0;
        }
        const uint32_t K = kk < hi - lo ? kk : hi - lo;
        uint64_t prev = 0;
        for (uint32_t u = 0; u < K; u++) {
            uint64_t best = ~0ull;
            for (uint32_t j = lo + (uint32_t)tid; j < hi; j += (uint32_t)nthr) {
                uint32_t ml;
                const uint64_t kj = t1 ? sm.key[j] : s1 ? (uint64_t)s1_pair(j, &ml) : key(j);
                if (kj > prev && kj < best) best = kj;
            }
            prev = k4s_min(best);
            if (tid == 0) sm.sel[u] = (uint32_t)(prev & (t1 ? 1023u : 4095u));
        }
        K4_SYNC();
        /* a T1 substitution is the nibble mask ML ^ runner-up at its byte */
        for (uint32_t u = (uint32_t)tid; u < K; u += (uint32_t)nthr) {
            const uint32_t j = sm.sel[u];
            sm.delta[u] = t1 ? k4s_delta(j / 2 - off, (uint32_t)((sm.mr[j] >> 4) ^ (sm.mr[j] & 15u)) << (j & 1u ? 0 : 4), blk - 2)
                        : s1 ? k4s_delta(j / 8 - off, 0x80u >> (j % 8), blk - 2)
                             : k4s_delta((j - 17) / 8 - off, 0x80u >> ((j - 17) % 8), blk - 2);
        }
        K4_SYNC();
        int64_t npass = 0;
        uint64_t first = ~0ull;
        for (uint32_t x = (uint32_t)tid; x < 64; x += (uint32_t)nthr) {
            if ((x == 0 && !t1 && !s1) || x >= (1u << K)) continue;     /* T1, S1: pattern 0 is pure ML */
            uint32_t s = syn;
            for (uint32_t u = 0; u < K; u++) if (x >> u & 1u) s ^= sm.delta[u];
            if (s == 0) { npass++; if (x < first) first = x; }
        }
        npass = k4s_sum(npass);
        first = k4s_min(first);
        if (npass != 1) { outcome = npass ? K4R_AMBIGUOUS : K4R_UNREPAIRABLE; break; }
        if (tid == 0)
            for (uint32_t u = 0; u < K; u++) {
                if (!(first >> u & 1u)) continue;
                const uint32_t j = sm.sel[u];
                if (t1) sm.pkt[j / 2] ^= (uint8_t)(((sm.mr[j] >> 4) ^ (sm.mr[j] & 15u)) << (j & 1u ? 0 : 4));
                else if (s1) sm.pkt[j / 8] ^= (uint8_t)(0x80u >> (j % 8));
                else sm.pkt[(j - 17) / 8] ^= (uint8_t)(0x80u >> ((j - 17) % 8));
            }
        K4_SYNC();
        if (t1) {                                               /* the symbols whose nibble differs from the hard decode */
            int64_t changed = 0;
            for (uint32_t i = lo + (uint32_t)tid; i < hi; i += (uint32_t)nthr)
                changed += sm.hard[i] != (i & 1u ? sm.pkt[i / 2] & 15u : sm.pkt[i / 2] >> 4);
            flips += (uint32_t)k4s_sum(changed);
        } else if (s1) {                                        /* the bits that differ from the hard decode */
            int64_t changed = 0;
            for (uint32_t q = lo + (uint32_t)tid; q < hi; q += (uint32_t)nthr) {
                const uint32_t x = WMB_BIT_DATA(b[1 + 2 * q]), c = WMB_BIT_DATA(b[2 + 2 * q]);
                changed += x == c || c != (uint32_t)(sm.pkt[q / 8] >> (7 - q % 8) & 1u);
            }
            flips += (uint32_t)k4s_sum(changed);
        } else flips += (uint32_t)wmb_popc((uint32_t)first);
        blocks++;
        K4_SYNC();
    }
    if (outcome == K4R_NONE) outcome = K4R_REPAIRED;
    r.outcome = (uint8_t)outcome;
    if (outcome != K4R_REPAIRED) { if (tid == 0) p.rep[lb + f] = r; return; }

    /* the repaired telegram: CRC-stripped datagram (format A :551-592, format B :595-636) into the pool */
    const uint32_t out_len = len - 2 * nblk;
    if (tid == 0) {
        const uint32_t room = (out_len + 3u) & ~3u;
        uint32_t o = k4_gadd(p.pool_n, room);
        if (o > p.pool_cap || room > p.pool_cap - o) {
#ifdef WMB_HOSTSIM
            *p.errors |= 8u;
#else
            atomicOr(p.errors, 8u);
#endif
            o = 0xFFFFFFFFu;
        }
        sm.data_off = o;
    }
    K4_SYNC();
    const uint32_t data_off = sm.data_off;
    if (data_off != 0xFFFFFFFFu)
        for (uint32_t i = (uint32_t)tid; i < out_len; i += (uint32_t)nthr)
            p.pool[data_off + i] = bframe ? (i == 0 ? (uint8_t)(sm.pkt[0] - 2 * nblk) : sm.pkt[wmb_strip_src_b(i)])
                                          : sm.pkt[wmb_strip_src_a(i)];
    if (tid == 0) {
        r.serial = (uint32_t)sm.pkt[4] | ((uint32_t)sm.pkt[5] << 8) | ((uint32_t)sm.pkt[6] << 16) | ((uint32_t)sm.pkt[7] << 24);
        r.data_off = data_off;
        r.len = (uint16_t)(data_off == 0xFFFFFFFFu ? 0 : out_len);
        r.erasures = (uint8_t)(flips < 255 ? flips : 255); r.blocks = (uint8_t)blocks;
        r.packet_rssi = (uint8_t)WMB_BIT_RSSI(b[1]);
        r.current_rssi = (uint8_t)WMB_BIT_RSSI(b[P - 1]);
        p.rep[lb + f] = r;
    }
}

/* wmb_reset: a new capture starts -- carried states, stream bookkeeping, gather state and error flags back to their
 * initial values, in stream order (no host copies, no synchronisation) */
struct ResetParams {
    IirState *ia_carry[WMB_N_CHAINS]; RlState *rl_carry[WMB_N_CHAINS];
    StreamDev *sd[WMB_N_STREAMS];
    GatherDev *gd; uint32_t *errors;                /* errors: 16 words (flags, per-pass fail counters, tile counter) */
};
WMB_D void wmb_reset_device(const ResetParams &p)
{
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (p.ia_carry[ch]) { IirState ia; iir_state_init(ia); *p.ia_carry[ch] = ia; }
        if (p.rl_carry[ch]) { RlState rl; rl_state_init(rl, ch); *p.rl_carry[ch] = rl; }
    }
    for (int k = 0; k < WMB_N_STREAMS; k++)
        if (p.sd[k]) { StreamDev z; z.total = 0; z.n_cand = 0; z.cand_overflow = 0; z.t2_sr = 0; z.pad = 0; *p.sd[k] = z; }
    GatherDev g;
    memset(&g, 0, sizeof(g));
    *p.gd = g;
    for (int i = 0; i < 16; i++) p.errors[i] = 0;
}
#ifdef WMB_HOSTSIM
/* ---- time2 blocks in the CPU build ----
 * The CPU launch runs a time2 kernel as one call per tile (k2t_count / k2t_write, the tile being the scans' lane): the
 * block's barrier-separated phases one after another over its threads, in the order hs_for picks.  Only the block scan
 * differs from the device's: serial over the threads' parts instead of warp shuffles. */
template <class F> static void hs_for(uint32_t n, F f);

/* exclusive scan, in place, of part[0..n) on top of `acc`; returns the inclusive total */
template <class CH>
static T2Fold t2_scan_serial(T2Fold *part, uint32_t n, T2Fold acc)
{
    for (uint32_t t = 0; t < n; t++) { const T2Fold f = part[t]; part[t] = acc; acc = t2_fold<CH>(acc, f); }
    return acc;
}
template <class CH>
static void k2t_count(const K2tParams &p, uint32_t tile)
{
    static T2Fold part[T2_THREADS];
    hs_for(T2_THREADS, [&](uint32_t t) { part[t] = k2t_load<CH>(p, tile, t, nullptr); });
    const T2Fold zero = { 0, 0, 0 };
    k2t_count_store(p, tile, t2_scan_serial<CH>(part, T2_THREADS, zero));
}
template <class CH>
static void k2t_write(const K2tParams &p, uint32_t tile)
{
    static T2Fold part[T2_THREADS];
    static K2tSmem sm;
    memset(&sm, 0xA5, sizeof(sm));                                     /* garbage-filled like real smem */
    hs_for(T2_THREADS, [&](uint32_t t) { part[t] = k2t_load<CH>(p, tile, t, &sm); });
    t2_scan_serial<CH>(part, T2_THREADS, k2t_carry<CH>(p, tile));
    hs_for(T2_THREADS, [&](uint32_t t) { k2t_spread<CH>(t, part[t], sm); });
    for (uint32_t r = 0; r < T2_WPT; r++) {
        hs_for(T2_THREADS, [&](uint32_t t) { k2t_emit<CH>(p, tile, t, r, sm); });
        hs_for(T2_THREADS, [&](uint32_t t) { k2t_flush(p, tile, t, r, sm); });
    }
}
#endif
#ifndef WMB_HOSTSIM
/* ---- __global__ wrappers ---- */
__global__ void __launch_bounds__(SCAN_BLOCK) cscan_a_kernel(const CountScan p)
{
    __shared__ uint64_t part[SCAN_BLOCK];
    cscan_local(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    if (threadIdx.x == 0) cscan_a_finish(p, blockIdx.x, part);
}
__global__ void cscan_b_kernel(const CountScan p) { if (threadIdx.x == 0 && blockIdx.x == 0) cscan_b(p); }
__global__ void __launch_bounds__(SCAN_BLOCK) cscan_c_kernel(const CountScan p)
{
    __shared__ uint64_t part[SCAN_BLOCK];
    cscan_local(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    if (threadIdx.x == 0) cscan_c_block(p, blockIdx.x, part);
    __syncthreads();
    cscan_c_write(p, blockIdx.x, threadIdx.x, part);
}
/* time2: exclusive scan of one T2Fold per thread, in thread order, on top of `carry` (the CPU build's k2t_count /
 * k2t_write below run it serially): a shuffle scan in every warp, the warps' totals through shared memory.  The inclusive total is the last
 * thread's result folded with its own value. */
template <class CH, int NT>
__device__ T2Fold t2_block_scan(const T2Fold v, const T2Fold carry, T2Fold (&wtot)[NT / 32])
{
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    T2Fold inc = v;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        T2Fold u;
        u.cnt = __shfl_up_sync(0xFFFFFFFFu, inc.cnt, o);
        u.tail = __shfl_up_sync(0xFFFFFFFFu, inc.tail, o);
        u.len = __shfl_up_sync(0xFFFFFFFFu, inc.len, o);
        if (lane >= o) inc = t2_fold<CH>(u, inc);
    }
    if (lane == 31) wtot[w] = inc;
    T2Fold ex;
    ex.cnt = __shfl_up_sync(0xFFFFFFFFu, inc.cnt, 1);
    ex.tail = __shfl_up_sync(0xFFFFFFFFu, inc.tail, 1);
    ex.len = __shfl_up_sync(0xFFFFFFFFu, inc.len, 1);
    __syncthreads();
    T2Fold acc = carry;
    for (uint32_t i = 0; i < w; i++) acc = t2_fold<CH>(acc, wtot[i]);
    return lane ? t2_fold<CH>(acc, ex) : acc;
}
template <class CH>
__global__ void __launch_bounds__(T2_THREADS) k2t_count_kernel(const K2tParams p)
{
    __shared__ T2Fold wtot[T2_THREADS / 32];
    const T2Fold f = k2t_load<CH>(p, blockIdx.x, threadIdx.x, nullptr);
    const T2Fold zero = { 0, 0, 0 };
    const T2Fold ex = t2_block_scan<CH, T2_THREADS>(f, zero, wtot);
    if (threadIdx.x == T2_THREADS - 1) k2t_count_store(p, blockIdx.x, t2_fold<CH>(ex, f));
}
template <class CH>
__global__ void __launch_bounds__(SCAN_BLOCK) t2scan_a_kernel(const K2tParams p)
{
    __shared__ T2Fold part[SCAN_BLOCK];
    t2scan_local<CH>(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    if (threadIdx.x == 0) t2scan_a_finish<CH>(p, blockIdx.x, part);
}
template <class CH>
__global__ void t2scan_b_kernel(const K2tParams p) { if (threadIdx.x == 0 && blockIdx.x == 0) t2scan_b<CH>(p); }
template <class CH>
__global__ void __launch_bounds__(SCAN_BLOCK) t2scan_c_kernel(const K2tParams p)
{
    __shared__ T2Fold part[SCAN_BLOCK];
    t2scan_local<CH>(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    if (threadIdx.x == 0) t2scan_c_block<CH>(p, blockIdx.x, part);
    __syncthreads();
    t2scan_c_write<CH>(p, blockIdx.x, threadIdx.x, part);
}
template <class CH>
__global__ void __launch_bounds__(T2_THREADS) k2t_write_kernel(const K2tParams p)
{
    __shared__ K2tSmem sm;
    __shared__ T2Fold wtot[T2_THREADS / 32];
    const T2Fold f = k2t_load<CH>(p, blockIdx.x, threadIdx.x, &sm);
    const T2Fold ex = t2_block_scan<CH, T2_THREADS>(f, k2t_carry<CH>(p, blockIdx.x), wtot);
    k2t_spread<CH>(threadIdx.x, ex, sm);
    __syncthreads();
    for (uint32_t r = 0; r < T2_WPT; r++) {
        k2t_emit<CH>(p, blockIdx.x, threadIdx.x, r, sm);
        __syncwarp();
        k2t_flush(p, blockIdx.x, threadIdx.x, r, sm);
        __syncwarp();                                             /* the next round reuses the staging */
    }
}
template <class CH>
__global__ void __launch_bounds__(K2_THREADS) k2a_lanes_kernel(const K2aParams p)
{
    k2a_lane<CH>(p, blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void k2a_verify_kernel(const K2aParams p, uint32_t *n_fail)
{
    k2a_verify_lane(p, blockIdx.x * blockDim.x + threadIdx.x, n_fail);
}
template <class CH>
__global__ void __launch_bounds__(K2_THREADS) k2m_lanes_kernel(const K2mParams p)
{
    k2m_lane<CH>(p, blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void k2m_verify_kernel(const K2mParams p, uint32_t *n_fail)
{
    k2m_verify_lane(p, blockIdx.x * blockDim.x + threadIdx.x, n_fail);
}
__global__ void __launch_bounds__(128) k2p1_lanes_kernel(const K2p1Params p) { k2p1_lane(p, blockIdx.x * blockDim.x + threadIdx.x); }
__global__ void k2p1_verify_kernel(const K2p1Params p, uint32_t *n_fail) { k2p1_verify_lane(p, blockIdx.x * blockDim.x + threadIdx.x, n_fail); }
__global__ void k2pc_compact_kernel(const K2pcParams p) { k2pc_compact(p, blockIdx.x, threadIdx.x, blockDim.x); }
__global__ void __launch_bounds__(128) k2p2_count_kernel(const K2p2Params p) { k2p2_count(p, blockIdx.x * blockDim.x + threadIdx.x); }
__global__ void __launch_bounds__(K2P2W_THREADS) k2p2_sum_kernel(const K2p2Params p)
{
    __shared__ uint32_t part[K2P2W_THREADS];
    k2p2w_a(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    if (threadIdx.x < 32) {                       /* warp 0 adds the block's partial sums */
        uint32_t s = 0;
        for (uint32_t t = threadIdx.x; t < K2P2W_THREADS; t += 32) s += part[t];
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, d);
        if (threadIdx.x == 0) p.cnt[blockIdx.x] = s;
    }
}
__global__ void __launch_bounds__(K2P2W_THREADS) k2p2_write_kernel(const K2p2Params p)
{
    __shared__ uint32_t part[K2P2W_THREADS];
    k2p2w_a(p, blockIdx.x, threadIdx.x, part);
    __syncthreads();
    k2p2w_b(part, threadIdx.x);
    __syncthreads();
    k2p2w_c(p, blockIdx.x, threadIdx.x, part);
}
__global__ void k2p_fold_kernel(const P1State *p1_end, RlState *p2_out, RlState *carry, const K2pDev *pd, const RlState *mono_end,
                                uint32_t *stat_fallbacks)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) k2p_fold(p1_end, p2_out, carry, pd, mono_end, stat_fallbacks);
}
__global__ void k2m_carry_kernel(const RlState *end, RlState *carry, const uint32_t *run_if)
{
    if (threadIdx.x == 0 && blockIdx.x == 0 && (!run_if || *run_if)) *carry = *end;
}

/* ---- lane verification without the host ------------------------------------------------------------------------
 * A speculative pass is followed by its verify kernel (every lane: start state == predecessor's end state?  count
 * the refuted ones) and by ONE block of the matching fix-up kernel: nothing to do in the common case (n_fail == 0,
 * a few microseconds); otherwise it re-runs the refuted lanes from their predecessors' exact end states and verifies
 * again until no lane is refuted -- what the host used to drive with a stream synchronisation per round. */
#define FIX_THREADS 128
/* Before that block: the same thing in parallel over segments of FIX_SEG lanes, one warp per segment (skipped when no
 * lane is refuted).  A clean carrier next to the channel leaves the clock filter near a fixed point between telegrams,
 * where two trajectories can stay an ulp apart for good: then whole runs of lanes are refuted (measured: every lane of
 * a five-carrier capture at noise sigma 4) and one block of 128 threads takes lanes / 128 lane times per round.  A
 * segment's warp iterates re-run + verify over its lanes until they are consistent with the segment's FIRST lane,
 * which it leaves alone (its predecessor belongs to another block).  Whatever this pass leaves behind -- refuted first
 * lanes, chains across segments -- the single block finds when it verifies every lane again: the pass is an
 * accelerator, the proof of exactness is still that block's "no lane refuted". */
#define FIX_SEG 32
template <class RERUN, class VERIFY>
__device__ __forceinline__ void fixup_segments(uint32_t lanes, const uint32_t *n_fail, const uint32_t *flags, uint32_t *stat_rerun,
                                               RERUN rerun, VERIFY verify)
{
    if (*(volatile const uint32_t *)n_fail == 0) return;
    __shared__ uint32_t s_cnt, s_dummy;
    const uint32_t l1 = min(lanes, (blockIdx.x + 1u) * FIX_SEG);
    const uint32_t lane = blockIdx.x * FIX_SEG + 1u + threadIdx.x;
    for (uint32_t round = 0; round < FIX_SEG; round++) {
        if (threadIdx.x == 0) { s_cnt = 0; s_dummy = 0; }
        __syncthreads();
        const bool flagged = lane < l1 && ((volatile const uint32_t *)flags)[lane] != 0;
        if (flagged) atomicAdd(&s_cnt, 1u);
        __syncthreads();
        const uint32_t n = s_cnt;
        if (n == 0) break;
        if (threadIdx.x == 0) atomicAdd(stat_rerun, n);
        if (flagged) rerun(lane);
        __threadfence();
        __syncthreads();
        if (lane < l1) verify(lane, &s_dummy);
        __threadfence();
        __syncthreads();
    }
}
template <class RERUN, class VERIFY>
__device__ __forceinline__ void fixup_loop(uint32_t lanes, uint32_t *n_fail, uint32_t *stat_rerun, uint32_t *errors,
                                           RERUN rerun, VERIFY verify)
{
    __shared__ uint32_t s_fail;
    /* the segment pass has changed lanes since the count was taken: count again */
    __syncthreads();
    if (threadIdx.x == 0) s_fail = *(volatile uint32_t *)n_fail;
    __syncthreads();
    if (s_fail == 0) return;
    __syncthreads();
    if (threadIdx.x == 0) *n_fail = 0;
    __threadfence();
    __syncthreads();
    for (uint32_t lane = threadIdx.x; lane < lanes; lane += blockDim.x) verify(lane);
    __threadfence();
    for (uint32_t round = 0;; round++) {
        __syncthreads();
        if (threadIdx.x == 0) s_fail = *(volatile uint32_t *)n_fail;
        __syncthreads();
        const uint32_t nf = s_fail;
        if (nf == 0) return;
        if (round > lanes + 2) {                                  /* cannot happen: lane 0 is exact, so every round fixes at least one lane */
            if (threadIdx.x == 0) { atomicOr(errors, 256u); *n_fail = 0; }
            return;
        }
        __syncthreads();
        if (threadIdx.x == 0) { atomicAdd(stat_rerun, nf); *n_fail = 0; }
        __threadfence();
        __syncthreads();
        for (uint32_t lane = threadIdx.x; lane < lanes; lane += blockDim.x) rerun(lane);      /* returns at once unless flagged */
        __threadfence();
        __syncthreads();
        for (uint32_t lane = threadIdx.x; lane < lanes; lane += blockDim.x) verify(lane);
        __threadfence();
    }
}
template <class CH>
__global__ void __launch_bounds__(FIX_THREADS) k2a_fixup_kernel(K2aParams p, uint32_t *n_fail, uint32_t *stat_rerun, uint32_t *errors)
{
    p.mode = 1;
    fixup_loop(p.lanes, n_fail, stat_rerun, errors, [&](uint32_t lane) { k2a_lane<CH>(p, lane); },
               [&](uint32_t lane) { k2a_verify_lane(p, lane, n_fail); });
}
template <class CH>
__global__ void __launch_bounds__(FIX_SEG) k2a_fixseg_kernel(K2aParams p, const uint32_t *n_fail, uint32_t *stat_rerun)
{
    p.mode = 1;
    fixup_segments(p.lanes, n_fail, p.rerun, stat_rerun, [&](uint32_t lane) { k2a_lane<CH>(p, lane); },
                   [&](uint32_t lane, uint32_t *cnt) { k2a_verify_lane(p, lane, cnt); });
}
template <class CH>
__global__ void __launch_bounds__(FIX_SEG) k2m_fixseg_kernel(K2mParams p, const uint32_t *n_fail, uint32_t *stat_rerun)
{
    p.mode = 1;
    fixup_segments(p.lanes, n_fail, p.rerun, stat_rerun, [&](uint32_t lane) { k2m_lane<CH>(p, lane); },
                   [&](uint32_t lane, uint32_t *cnt) { k2m_verify_lane(p, lane, cnt); });
}
__global__ void __launch_bounds__(FIX_SEG) k2p1_fixseg_kernel(K2p1Params p, const uint32_t *n_fail, uint32_t *stat_rerun)
{
    p.mode = 1;
    fixup_segments(p.lanes, n_fail, p.rerun, stat_rerun, [&](uint32_t lane) { k2p1_lane(p, lane); },
                   [&](uint32_t lane, uint32_t *cnt) { k2p1_verify_lane(p, lane, cnt); });
}
template <class CH>
__global__ void __launch_bounds__(FIX_THREADS) k2m_fixup_kernel(K2mParams p, uint32_t *n_fail, uint32_t *stat_rerun, uint32_t *errors)
{
    p.mode = 1;
    fixup_loop(p.lanes, n_fail, stat_rerun, errors, [&](uint32_t lane) { k2m_lane<CH>(p, lane); },
               [&](uint32_t lane) { k2m_verify_lane(p, lane, n_fail); });
}
__global__ void __launch_bounds__(FIX_THREADS) k2p1_fixup_kernel(K2p1Params p, uint32_t *n_fail, uint32_t *stat_rerun, uint32_t *errors)
{
    p.mode = 1;
    fixup_loop(p.lanes, n_fail, stat_rerun, errors, [&](uint32_t lane) { k2p1_lane(p, lane); },
               [&](uint32_t lane) { k2p1_verify_lane(p, lane, n_fail); });
}
__global__ void k2c_compact_kernel(const K2cParams p) { k2c_compact(p, blockIdx.x, threadIdx.x, blockDim.x); }
__global__ void wmb_reset_kernel(const ResetParams p) { if (threadIdx.x == 0 && blockIdx.x == 0) wmb_reset_device(p); }

/* test hook (wmb_debug_arith): the device arithmetic on caller-made operands */
__global__ void dbg_arith_kernel(const float *y, const float *x, float *out, size_t n, int mode)
{
    __shared__ WmbAtanTab tab;
    wmb_atan_tab_fill(&tab, (int)threadIdx.x);
    __syncthreads();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float r;
        if (mode == 0) r = wmb_atan2f_bounded(y[i], x[i], &tab);
        else if (mode == 1) r = wmb_atan2f(y[i], x[i]);
        else if (mode == 2) r = wmb_fdiv_bounded(y[i], x[i]);
        else if (mode == 3) r = wmb_fsqrt_pos(y[i]);
        else r = wmb_discriminator(y[i], x[i], y[i ? i - 1 : 0], x[i ? i - 1 : 0], &tab);
        out[i] = r;
    }
}
__global__ void k3_plan_kernel(const K3Params p) { if (threadIdx.x == 0 && blockIdx.x == 0) k3_plan(p); }
__global__ void k3_publish_kernel(const K3Params p) { if (threadIdx.x == 0 && blockIdx.x == 0) k3_publish(p); }
/* the kernels below do not know on the host how many candidates there are: grid-stride loops over gd->n */
#define K3_FILL_PARTS 8
__global__ void k3_fill_kernel(const K3Params p)
{
    /* all threads of a warp stay in the loop together (the shuffles inside k3_fill need them): whole groups of 8 */
    const uint32_t n = p.gd->n, stride = gridDim.x * blockDim.x / K3_FILL_PARTS;
    const uint32_t n_pad = (n + 3u) & ~3u;                       /* 4 candidates per warp */
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) / K3_FILL_PARTS; i < n_pad; i += stride)
        k3_fill(p, i, threadIdx.x % K3_FILL_PARTS, K3_FILL_PARTS);
}
__global__ void k3_size_kernel(const K3Params p)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.gd->n; i += gridDim.x * blockDim.x) k3_size(p, i);
}
__global__ void k3_cut_kernel(const K3Params p)
{
    for (uint32_t i = blockIdx.x; i < p.gd->n; i += gridDim.x) k3_cut(p, i, threadIdx.x, blockDim.x);
}
__global__ void __launch_bounds__(SCAN_THREADS) k3_offsets_kernel(const K3Params p)
{
    k3_offsets_a(p, threadIdx.x);
    __syncthreads();
    if (threadIdx.x == 0) k3_offsets_b(p);
    __syncthreads();
    k3_offsets_c(p, threadIdx.x);
}
__global__ void k3_soft_kernel(const K3Params p)
{
    for (uint32_t i = blockIdx.x; i < p.gd->n; i += gridDim.x) k3_soft<false>(p, i, threadIdx.x, blockDim.x);
}
__global__ void k3_soft_s1_kernel(const K3Params p)
{
    for (uint32_t i = blockIdx.x; i < p.gd->n; i += gridDim.x) k3_soft<true>(p, i, threadIdx.x, blockDim.x);
}
__global__ void k3_copy_kernel(const K3Params p)
{
    for (uint32_t i = blockIdx.x; i < p.gd->n; i += gridDim.x) k3_copy(p, i, threadIdx.x, blockDim.x);
}
__global__ void k3_carry_kernel(const K3Params p)
{
    const uint32_t n = p.gd->n > WMB_N_STREAMS ? p.gd->n : WMB_N_STREAMS;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) k3_carry(p, i);
}
__global__ void __launch_bounds__(K4_THREADS) k4_decode_kernel(const K4Params p)
{
    __shared__ K4Smem sm;
    const uint32_t n = k4_count(p);
    for (uint32_t f = blockIdx.x; f < n; f += gridDim.x) {
        k4_decode(p, f, threadIdx.x, blockDim.x, sm);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(K4_THREADS) k4r_repair_kernel(const K4RParams p)
{
    __shared__ K4RSmem sm;
    const uint32_t n = k4r_count(p);
    for (uint32_t f = blockIdx.x; f < n; f += gridDim.x) {
        k4r_repair(p, f, threadIdx.x, blockDim.x, sm);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(K4_THREADS) k4s_repair_kernel(const K4SParams p)
{
    __shared__ K4SSmem sm;
    const uint32_t n = k4s_count(p);
    for (uint32_t f = blockIdx.x; f < n; f += gridDim.x) {
        k4s_repair<false>(p, f, threadIdx.x, blockDim.x, sm);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(K4_THREADS) k4s_s1_repair_kernel(const K4SParams p)
{
    __shared__ K4SSmem sm;
    const uint32_t n = k4s_count(p);
    for (uint32_t f = blockIdx.x; f < n; f += gridDim.x) {
        k4s_repair<true>(p, f, threadIdx.x, blockDim.x, sm);
        __syncthreads();
    }
}
#endif
