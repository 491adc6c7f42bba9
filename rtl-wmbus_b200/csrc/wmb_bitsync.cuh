/*
 * wmb_bitsync.cuh -- K2: the sequential recurrences of a receiver chain, restructured
 * for the GPU.  (A single "everything per lane" kernel was dominated by divergence, because
 * a float recurrence, a branchy integer state machine and event output shared one loop.)
 *
 *   K2a  k2a_lane      float-only lanes: [DC block] -> slicer bit, x^2 -> 3 biquads ->
 *                      clock sign -> lock stencil.  Writes bit-packed streams per
 *                      decimated sample: sbits (time2 strobe) and, with -o, dbits (data
 *                      bit; without the DC block the demod kernel K1 slices them).
 *                      Speculative warm-up + state verification (rtl_wmbus.c:497-515,
 *                      :1059, :1089-1111; iir.h:59-74).
 *   K2t  k2t_*         time2 bit stream: strobed data bits -> shift register -> access
 *                      code.  Exact without speculation: each tile of words reports its
 *                      strobe count and its last 24 strobed bits, a scan folds them into
 *                      every tile's start register (rtl_wmbus.c:806-852).
 *   K2m  k2m_lane      run-length bit sync, integer-only lanes reading dbits
 *                      (rtl_wmbus.c:617-803).  Speculative warm-up + verification.
 */
#pragma once
#include "wmb_exact.cuh"
#include "wmb_chain.cuh"

struct u32x4 { uint32_t x, y, z, w; };

/* ------------------------------------------------------------------------------------- */
/* K2a: clock-recovery lanes                                                             */
/* ------------------------------------------------------------------------------------- */

struct K2aParams {
    const float *dphi;          /* index 0 = batch sample 0; [-hist, M) readable              */
    int64_t  M, hist;
    uint32_t C, W, lanes;       /* all multiples of 32                                        */
    uint32_t *dbits, *sbits;    /* word w covers samples 32w..32w+31 (bit i = sample 32w+i); dbits written with -o only:
                                   without the DC block the demod kernel slices them                */
    uint32_t *cbits;            /* optional stage tap: the clock signs (null unless the context was made with taps) */
    IirState *st_start, *st_end;
    const IirState *carry;
    uint32_t *rerun;
    uint32_t mode;              /* 0 speculative pass, 1 re-run flagged lanes                 */
    uint32_t dc, t2;            /* -o ; time2 enabled (else only the data bits are produced)  */
    uint32_t spec0;             /* lane 0 starts cold from the history too (its predecessor -- the previous batch's last
                                   lane -- may still be running); verified against the carried state like any lane  */
    uint32_t lock;              /* clock-lock threshold L, 1..WMB_LOCK_MAX (wmb_set_receiver)                  */
};

/* registers of one clock-recovery lane */
struct K2aRegs {
    float dcx, dcy;
    float h10, h20, h11, h21, h12, h22;
    uint32_t clk3;
};

/* 32 decimated samples (one 128-byte line of dphi, already in registers) through the DC block,
 * the slicer and the three biquads; returns the data-bit and clock-sign words */
template <class CH, bool dc, bool t2, bool warm>
WMB_D void k2a_block(const float4 (&blk)[8], int n, K2aRegs &r, uint32_t &dword, uint32_t &cword)
{
    constexpr float b10 = CH::B10, b20 = CH::B20, a10 = CH::A10, a20 = CH::A20;
    constexpr float b11 = CH::B11, b21 = CH::B21, a11 = CH::A11, a21 = CH::A21;
    constexpr float b12 = CH::B12, b22 = CH::B22, a12 = CH::A12, a22 = CH::A22;
    constexpr float gain = 1.874981046e-06;                       /* rtl_wmbus.c:338 */
    constexpr float alpha = 0.999f, cdc = (1.f + 0.999f) / 2.f;   /* rtl_wmbus.c:501 / :511 */
    dword = 0; cword = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) {
        if (i >= n) break;
        const float4 q = blk[i >> 2];
        float x = (i & 3) == 0 ? q.x : (i & 3) == 1 ? q.y : (i & 3) == 2 ? q.z : q.w;
        if (dc) {
            const float y = wmb_fadd(wmb_fmul(cdc, wmb_fsub(x, r.dcx)), wmb_fmul(alpha, r.dcy));
            r.dcx = x; r.dcy = y; x = y;
        }
        if (!warm) dword |= (x >= 0.0f ? 1u : 0u) << i;           /* rtl_wmbus.c:1059 */
        if (t2) {
            float v = wmb_fmul(x, x);                             /* rtl_wmbus.c:1089 */
            float h0;
            h0 = wmb_fsub(v, wmb_fadd(wmb_fmul(a10, r.h10), wmb_fmul(a20, r.h20)));
            v = wmb_fadd(wmb_fadd(h0, wmb_fmul(b10, r.h10)), wmb_fmul(b20, r.h20));
            r.h20 = r.h10; r.h10 = h0;
            h0 = wmb_fsub(v, wmb_fadd(wmb_fmul(a11, r.h11), wmb_fmul(a21, r.h21)));
            v = wmb_fadd(wmb_fadd(h0, wmb_fmul(b11, r.h11)), wmb_fmul(b21, r.h21));
            r.h21 = r.h11; r.h11 = h0;
            h0 = wmb_fsub(v, wmb_fadd(wmb_fmul(a12, r.h12), wmb_fmul(a22, r.h22)));
            /* a warm-up block only has to carry the state forward: the last section's output,
             * the gain and the two comparisons are not part of it (only the final three clock
             * signs are, and the block before the chunk start is computed in full) */
            if (!warm) {
                v = wmb_fadd(wmb_fadd(h0, wmb_fmul(b12, r.h12)), wmb_fmul(b22, r.h22));
                v = wmb_fmul(v, gain);
                cword |= (v >= 0.0f ? 1u : 0u) << i;
            }
            r.h22 = r.h12; r.h12 = h0;
        }
    }
}

/* The same arithmetic for a full block of 32 samples, software-pipelined across the cascade: in
 * step t the DC block works on sample t, the first biquad on sample t - o1, the second on t - o2
 * and the third on t - o3.  Every sample still sees exactly the operations of k2a_block in the
 * same order (the results are bit-identical); only independent work of neighbouring samples is
 * now adjacent in the instruction stream, which a single in-order warp needs to keep the FP pipe
 * busy (one sample alone is a chain of ~10 dependent 4-cycle operations). */
template <class CH, bool dc, bool t2>
WMB_D void k2a_block32(const float4 (&blk)[8], K2aRegs &r, uint32_t &dword, uint32_t &cword)
{
    constexpr float b10 = CH::B10, b20 = CH::B20, a10 = CH::A10, a20 = CH::A20;
    constexpr float b11 = CH::B11, b21 = CH::B21, a11 = CH::A11, a21 = CH::A21;
    constexpr float b12 = CH::B12, b22 = CH::B22, a12 = CH::A12, a22 = CH::A22;
    constexpr float gain = 1.874981046e-06;
    constexpr float alpha = 0.999f, cdc = (1.f + 0.999f) / 2.f;
    constexpr int o1 = dc ? 1 : 0, o2 = o1 + 1, o3 = o2 + 1;
    constexpr int steps = t2 ? 32 + o3 : 32;
    dword = 0; cword = 0;
    float q0 = 0.f, q1 = 0.f, q2 = 0.f;      /* pipeline registers between the stages */
#pragma unroll
    for (int t = 0; t < steps; t++) {
        if (t2 && t >= o3 && t - o3 < 32) {
            const float h0 = wmb_fsub(q2, wmb_fadd(wmb_fmul(a12, r.h12), wmb_fmul(a22, r.h22)));
            float v = wmb_fadd(wmb_fadd(h0, wmb_fmul(b12, r.h12)), wmb_fmul(b22, r.h22));
            v = wmb_fmul(v, gain);
            cword |= (v >= 0.0f ? 1u : 0u) << (t - o3);
            r.h22 = r.h12; r.h12 = h0;
        }
        if (t2 && t >= o2 && t - o2 < 32) {
            const float h0 = wmb_fsub(q1, wmb_fadd(wmb_fmul(a11, r.h11), wmb_fmul(a21, r.h21)));
            q2 = wmb_fadd(wmb_fadd(h0, wmb_fmul(b11, r.h11)), wmb_fmul(b21, r.h21));
            r.h21 = r.h11; r.h11 = h0;
        }
        if (t2 && t >= o1 && t - o1 < 32) {
            float x;
            if (dc) x = q0;
            else {
                const float4 q = blk[t >> 2];
                x = (t & 3) == 0 ? q.x : (t & 3) == 1 ? q.y : (t & 3) == 2 ? q.z : q.w;
            }
            const float v = wmb_fmul(x, x);
            const float h0 = wmb_fsub(v, wmb_fadd(wmb_fmul(a10, r.h10), wmb_fmul(a20, r.h20)));
            q1 = wmb_fadd(wmb_fadd(h0, wmb_fmul(b10, r.h10)), wmb_fmul(b20, r.h20));
            r.h20 = r.h10; r.h10 = h0;
        }
        if (t < 32) {
            const float4 q = blk[t >> 2];
            float x = (t & 3) == 0 ? q.x : (t & 3) == 1 ? q.y : (t & 3) == 2 ? q.z : q.w;
            if (dc) {
                const float y = wmb_fadd(wmb_fmul(cdc, wmb_fsub(x, r.dcx)), wmb_fmul(alpha, r.dcy));
                r.dcx = x; r.dcy = y; x = y;
                q0 = y;
            }
            dword |= (x >= 0.0f ? 1u : 0u) << t;
        }
    }
}

/* Clock lock on a whole word (rtl_wmbus.c:1092-1111): counting clock samples from a rising edge, the reference
 * delivers the data bit on the L-th high sample after it (opts_CLOCK_LOCK_THRESHOLD_*, :865-866), i.e. on sample m iff
 * the clock read low at m-L-1 and high at m-L..m.  `clk` holds the L+1 clock signs before the word, newest in bit 0
 * (zero before the stream's first sample: the clock reads low there).  LK = 2: the reference's threshold as a
 * constant, the default path; LK = 0: L from the launch, without a branch. */
template <int LK>
WMB_D uint32_t lock_strobes(uint32_t clk, uint32_t cword, uint32_t L)
{
    if (LK == 2) {
        const uint64_t hist3 = ((clk & 1u) << 2) | (clk & 2u) | ((clk >> 2) & 1u);   /* bit2 = m-1 */
        const uint64_t H = ((uint64_t)cword << 3) | hist3;
        return (uint32_t)((H >> 3) & (H >> 2) & (H >> 1) & ~H);
    }
    /* time order: bit L+1+i = sample i of the word, bit j = sample j-L-1 for j <= L */
    const uint64_t H = ((uint64_t)cword << (L + 1)) | (wmb_brev(clk) >> (31 - L));
    uint64_t high = H >> 1;
#pragma unroll
    for (uint32_t j = 2; j <= WMB_LOCK_MAX + 1; j++) high &= (j <= L + 1) ? (H >> j) : ~0ull;
    return (uint32_t)(high & ~H);
}

/* the clock history after a word of n samples (bits 0..n-1 of cword; none above) */
template <int LK>
WMB_D uint32_t lock_history(uint32_t clk, uint32_t cword, int n, uint32_t L)
{
    if (LK == 2) {
        if (n == 32) return ((cword >> 31) & 1u) | (((cword >> 30) & 1u) << 1) | (((cword >> 29) & 1u) << 2);
        for (int i = 0; i < n; i++) clk = ((clk << 1) | ((cword >> i) & 1u)) & 7u;
        return clk;
    }
    const uint32_t mask = (2u << L) - 1u, r = wmb_brev(cword);      /* r: bit k = sample 31 - k */
    return (n == 32 ? r : (clk << n) | (r >> (32 - n))) & mask;
}

WMB_D void k2a_load(float4 (&blk)[8], const float *src)
{
    const float4 *s4 = (const float4 *)src;
#pragma unroll
    for (int j = 0; j < 8; j++) blk[j] = s4[j];
}

WMB_D void k2a_save(IirState &st, const K2aRegs &r)
{
    st.dc_x = r.dcx; st.dc_y = r.dcy;
    st.h[0] = r.h10; st.h[1] = r.h20; st.h[2] = r.h11; st.h[3] = r.h21; st.h[4] = r.h12; st.h[5] = r.h22;
    st.clk3 = r.clk3; st.pad = 0;
}

#define K2A_L2_AHEAD 16

template <class CH, bool DC, bool T2, int LK>
WMB_D void k2a_lane_t(const K2aParams &p, uint32_t lane)
{
    if (lane >= p.lanes) return;
    const int64_t s0 = (int64_t)lane * p.C;
    const int64_t e0 = (s0 + p.C < p.M) ? s0 + p.C : p.M;
    IirState st;
    int64_t m;
    if (p.mode == 0) {
        if (lane == 0 && !p.spec0) { st = *p.carry; m = 0; }
        else {
            iir_state_init(st);
            m = s0 - (int64_t)p.W;
            if (m < -p.hist) m = -p.hist;
        }
    } else {
        if (!p.rerun[lane]) return;
        st = lane ? p.st_end[lane - 1] : *p.carry;
        m = s0;
    }
    K2aRegs r;
    r.dcx = st.dc_x; r.dcy = st.dc_y;
    r.h10 = st.h[0]; r.h20 = st.h[1]; r.h11 = st.h[2]; r.h21 = st.h[3]; r.h12 = st.h[4]; r.h22 = st.h[5];
    r.clk3 = st.clk3;
    bool saved_start = false;

    /* each lane streams whole 128-byte lines of dphi; a line is requested two blocks before it is
     * processed so that the DRAM latency under load hides behind ~64 recurrence steps
     * (reads may run up to 32 samples past the lane's end: the buffers carry that slack) */
    float4 cur[8], nxt[8], nx2[8];
    if (m < e0) k2a_load(cur, p.dphi + m);
    if (m + 32 < e0) k2a_load(nxt, p.dphi + m + 32);
    while (m < e0) {
        if (m + 64 < e0) k2a_load(nx2, p.dphi + m + 64);        /* two lines ahead: ~2 us of recurrence steps */
#ifndef WMB_HOSTSIM
        /* and the line 16 blocks ahead is pulled into L2 (no register cost), so that the register loads above
         * see L2 latency even when DRAM is busy with the other 18 k lanes */
        if (m + 32 * K2A_L2_AHEAD < e0) asm volatile("prefetch.global.L2 [%0];" :: "l"(p.dphi + m + 32 * K2A_L2_AHEAD));
#endif
        if (m == s0 && !saved_start) { k2a_save(st, r); p.st_start[lane] = st; saved_start = true; }
        const int n = (e0 - m >= 32) ? 32 : (int)(e0 - m);
        uint32_t dword, cword;
        /* (a variant that skips the output-only arithmetic during the warm-up was measured slower:
         * two 20 KB unrolled bodies thrash the instruction cache) */
        if (n == 32) k2a_block32<CH, DC, T2>(cur, r, dword, cword);
        else k2a_block<CH, DC, T2, false>(cur, n, r, dword, cword);
        const uint32_t sword = lock_strobes<LK>(r.clk3, cword, p.lock);
        r.clk3 = lock_history<LK>(r.clk3, cword, n, p.lock);
        if (m >= s0) {
            const uint32_t keep = (n == 32) ? 0xFFFFFFFFu : ((1u << n) - 1u);
            if (DC) p.dbits[m >> 5] = dword & keep;
            p.sbits[m >> 5] = sword & keep;
            if (p.cbits) p.cbits[m >> 5] = cword & keep;
        }
        m += n;
#pragma unroll
        for (int j = 0; j < 8; j++) { cur[j] = nxt[j]; nxt[j] = nx2[j]; }
    }
    k2a_save(st, r);
    if (!saved_start) p.st_start[lane] = st;                      /* empty lane */
    p.st_end[lane] = st;
}

template <class CH>
WMB_D void k2a_lane(const K2aParams &p, uint32_t lane)
{
    if (!p.t2) { if (p.dc) k2a_lane_t<CH, true, false, 2>(p, lane); else k2a_lane_t<CH, false, false, 2>(p, lane); }
    else if (p.lock == 2) { if (p.dc) k2a_lane_t<CH, true, true, 2>(p, lane); else k2a_lane_t<CH, false, true, 2>(p, lane); }
    else { if (p.dc) k2a_lane_t<CH, true, true, 0>(p, lane); else k2a_lane_t<CH, false, true, 0>(p, lane); }
}

#ifndef WMB_HOSTSIM
/* ------------------------------------------------------------------------------------- */
/* K2a, warp-cooperative: three threads per lane, one per biquad section                 */
/*                                                                                       */
/* k2a_lane_t above runs one lane per thread: ~38 instructions per sample on a single     */
/* dependent stream, 59 cycles per sample for a lone warp -- the lane's LENGTH in time is  */
/* what every small batch and every tail waits for, and it forces short lanes (many of    */
/* them, each with its own 24576-sample warm-up: 2.7 x redundant arithmetic at 1 GiB).    */
/* Here the three sections of a lane sit in three neighbouring threads and work on        */
/* different samples at the same moment: in step s thread r handles sample s - SKEW r,      */
/* takes its input from its left neighbour's output of SKEW steps ago (a shuffle issued    */
/* SKEW - 1 steps ahead: with one step of slack the warp measurably waits for it, 41       */
/* cycles per step), and the warp issues ONE biquad per step                               */
/* for ten lanes.  Every sample still sees exactly the operations of k2a_block in the     */
/* same order -- only the interleaving changes -- so states and bits are bit-identical to  */
/* the per-thread version (which stays: -o, re-runs, ragged final batches, CPU tests).    */
/* A step costs ~15 issue slots instead of 38 and its critical path is the biquad         */
/* recurrence itself (multiply, add, subtract: 12 cycles).                                */
/*                                                                                       */
/* All lanes of a warp run the same number of steps: W warm-up samples (lanes whose        */
/* warm-up is cut short by the start of the stream are fed zeros before it, which keeps a  */
/* zero state zero), C live samples, and one more block in which the two lagging sections */
/* reach the lane's end.  A lane's state "at sample q" is picked up section by section as  */
/* each thread arrives there (steps q, q+2, q+4).  Output bits are collected at the step's */
/* position in the block and re-aligned by 2r with a funnel shift when the next block is   */
/* complete (2 SKEW <= 31: a section's lag stays inside one block).                       */
/* ------------------------------------------------------------------------------------- */
#define K2A2_LPW 10                  /* lanes per warp: 30 threads, two idle */
#ifndef K2A2_THREADS
#define K2A2_THREADS 64
#endif

#ifndef K2A2_SKEW
#define K2A2_SKEW 6                  /* steps between a section and the next one (>= 2): the shuffle that carries a
                                        section's output to its neighbour has SKEW - 1 steps to arrive */
#endif

struct K2a2Thread {
    float h1, h2;                   /* this section's memories                                  */
    float o, sh[K2A2_SKEW - 1];     /* last output (to be passed on), shuffled inputs on their way (sh[0]: this step's) */
    float a1, a2, b1, b2;
    uint32_t R, Rprev;              /* bits of this block / the block before, at step positions */
    bool r0, r2;
};

template <bool OUT>
__device__ __forceinline__ void k2a2_step(K2a2Thread &t, const float xs, const int i)
{
    constexpr float gain = 1.874981046e-06;                       /* rtl_wmbus.c:338 */
    const float xx = wmb_fmul(xs, xs);                            /* rtl_wmbus.c:1089 */
    const float in = t.r0 ? xx : t.sh[0];
#pragma unroll
    for (int k = 0; k + 1 < K2A2_SKEW - 1; k++) t.sh[k] = t.sh[k + 1];
    t.sh[K2A2_SKEW - 2] = __shfl_up_sync(0xFFFFFFFFu, t.o, 1);    /* the neighbour's output of the step before: input SKEW - 1 steps from now */
    const float h0 = wmb_fsub(in, wmb_fadd(wmb_fmul(t.a1, t.h1), wmb_fmul(t.a2, t.h2)));
    const float out = wmb_fadd(wmb_fadd(h0, wmb_fmul(t.b1, t.h1)), wmb_fmul(t.b2, t.h2));
    t.h2 = t.h1; t.h1 = h0; t.o = out;
    if (OUT) {
        /* clock sign (only the last section's bits are kept; the data bits come from the demod kernel) */
        if (wmb_fmul(out, gain) >= 0.0f) t.R |= 1u << i;
    }
}

template <class CH, int LK>
__global__ void __launch_bounds__(K2A2_THREADS) k2a2_lanes_kernel(const K2aParams p)
{
    const int lid = threadIdx.x & 31;
    const int role = lid % 3;
    const uint32_t lane = (blockIdx.x * (K2A2_THREADS / 32) + (threadIdx.x >> 5)) * K2A2_LPW + lid / 3;
    const bool valid = lid < 3 * K2A2_LPW && lane < p.lanes;
    K2a2Thread t;
    t.h1 = t.h2 = t.o = 0.0f;
#pragma unroll
    for (int k = 0; k < K2A2_SKEW - 1; k++) t.sh[k] = 0.0f;
    t.R = t.Rprev = 0;
    t.r0 = role == 0; t.r2 = role == 2;
    t.a1 = role == 0 ? CH::A10 : role == 1 ? CH::A11 : CH::A12;
    t.a2 = role == 0 ? CH::A20 : role == 1 ? CH::A21 : CH::A22;
    t.b1 = role == 0 ? CH::B10 : role == 1 ? CH::B11 : CH::B12;
    t.b2 = role == 0 ? CH::B20 : role == 1 ? CH::B21 : CH::B22;

    const int64_t s0 = (int64_t)lane * p.C;
    const int64_t e0 = (s0 + p.C < p.M) ? s0 + p.C : p.M;
    const int64_t m0 = s0 - (int64_t)p.W;                           /* nominal start of the run; real samples begin at -hist */
    const int jw = (int)(p.W / 32);                                 /* first live block                                      */
    const int je = valid ? jw + (int)((e0 - s0) / 32) : -1;         /* block in which the sections reach the lane's end       */
    const int nb = jw + (int)(p.C / 32) + 1;                        /* blocks run by every lane of the grid                   */
    const int64_t m_last = p.M + 256;                               /* reads stay inside the buffer's slack                   */
    const bool loader = valid && t.r0;

    float4 cur[8], nxt[8];
    auto load = [&](float4 (&b)[8], int j) {
        const int64_t m = m0 + 32 * (int64_t)j;
        if (loader && m >= -p.hist) {
            const float4 *s4 = (const float4 *)(p.dphi + (m < m_last ? m : m_last));
#pragma unroll
            for (int q = 0; q < 8; q++) b[q] = s4[q];
            if (m + 32 * K2A_L2_AHEAD < p.M) asm volatile("prefetch.global.L2 [%0];" :: "l"(p.dphi + m + 32 * K2A_L2_AHEAD));
        } else {
#pragma unroll
            for (int q = 0; q < 8; q++) b[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
#define K2A2_X(i) ((i & 3) == 0 ? cur[i >> 2].x : (i & 3) == 1 ? cur[i >> 2].y : (i & 3) == 2 ? cur[i >> 2].z : cur[i >> 2].w)

    load(cur, 0);
    int j = 0;
    /* warm-up blocks but the last: state only */
    for (; j < jw - 1; j++) {
        load(nxt, j + 1);
#pragma unroll
        for (int i = 0; i < 32; i++) k2a2_step<false>(t, K2A2_X(i), i);
#pragma unroll
        for (int q = 0; q < 8; q++) cur[q] = nxt[q];
    }
    /* last warm-up block, live blocks, one block past the end: bits, states at the chunk borders, stores */
    uint32_t clk3 = 0;
    const int shr = K2A2_SKEW * role;                              /* this section's lag in samples */
    for (; j < nb; j++) {
        load(nxt, j + 1);
        const bool at_start = valid && j == jw, at_end = j == je;
        float c1 = 0.f, c2 = 0.f;
        t.R = 0;
#pragma unroll
        for (int i = 0; i < 32; i++) {
            if (i == 0 || i == K2A2_SKEW || i == 2 * K2A2_SKEW) {       /* section i / SKEW arrives at the block's first sample */
                if ((at_start || at_end) && role == i / K2A2_SKEW) { c1 = t.h1; c2 = t.h2; }
            }
            k2a2_step<true>(t, K2A2_X(i), i);
        }
        /* the block before this one is complete now: its samples sit 2r positions up */
        const uint32_t A = __funnelshift_r(t.Rprev, t.R, shr);
        t.Rprev = t.R;
        const int jb = j - 1;
        uint32_t sword = 0;
        if (t.r2) {
            sword = lock_strobes<LK>(clk3, A, p.lock);
            clk3 = lock_history<LK>(clk3, A, 32, p.lock);
            if (j == jw && m0 + 32 * (int64_t)jw <= -p.hist) clk3 = 0;     /* the lane starts at the stream's first sample: no clock history */
        }
        if (valid && jb >= jw && jb < je) {
            const int64_t w = (m0 >> 5) + jb;                               /* word of the batch (m0 is a multiple of 32) */
            if (t.r2) { p.sbits[w] = sword; if (p.cbits) p.cbits[w] = A; }
        }
        if (at_start || at_end) {
            IirState *st = at_end ? p.st_end + lane : p.st_start + lane;
            st->h[2 * role] = c1; st->h[2 * role + 1] = c2;
            if (t.r0) { st->dc_x = 0.f; st->dc_y = 0.f; }
            if (t.r2) { st->clk3 = clk3; st->pad = 0; }
            /* a lane without live samples (e0 == s0 cannot happen: lanes = ceil(M / C)) would need both at once */
        }
#pragma unroll
        for (int q = 0; q < 8; q++) cur[q] = nxt[q];
    }
#undef K2A2_X
}
#endif /* !WMB_HOSTSIM */

WMB_D bool iir_state_equal(const IirState &a, const IirState &b, uint32_t dc, uint32_t t2)
{
    bool eq = true;
    if (dc) eq = eq && wmb_f2u(a.dc_x) == wmb_f2u(b.dc_x) && wmb_f2u(a.dc_y) == wmb_f2u(b.dc_y);
    if (t2) {
        for (int i = 0; i < 6; i++) eq = eq && wmb_f2u(a.h[i]) == wmb_f2u(b.h[i]);
        eq = eq && a.clk3 == b.clk3;                 /* the L+1 signs the lock stencil reads, no other bit is set */
    }
    return eq;
}

WMB_D void k2a_verify_lane(const K2aParams &p, uint32_t lane, uint32_t *n_fail)
{
    if (lane >= p.lanes) return;
    uint32_t bad = 0;
    if (lane > 0) { if (!iir_state_equal(p.st_start[lane], p.st_end[lane - 1], p.dc, p.t2)) bad = 1; }
    else if (p.spec0 && !iir_state_equal(p.st_start[0], *p.carry, p.dc, p.t2)) bad = 1;
    p.rerun[lane] = bad;
    if (bad) {
#ifdef WMB_HOSTSIM
        (*n_fail)++;
#else
        atomicAdd(n_fail, 1u);
#endif
    }
}

/* ------------------------------------------------------------------------------------- */
/* K2t: time2 bit stream                                                                 */
/* ------------------------------------------------------------------------------------- */

/* access-code match with up to `errors` bit errors: count_set_bits((bitstream & MASK) ^ CODE) <= ERRORS (rtl_wmbus.c:688,
 * :773, :822, :846; ACCESS_CODE_*_ERRORS, :99, :103) */
template <class CH>
WMB_D uint32_t ac_match(uint32_t sr, uint32_t errors)
{
    return (uint32_t)wmb_popc((sr & CH::CODE_MASK) ^ CH::CODE) <= errors ? 1u : 0u;
}

struct StreamDev {                  /* device-resident bookkeeping of one (chain, algo) stream */
    uint64_t total;                 /* events appended so far (== next ordinal)            */
    uint32_t n_cand;                /* candidates collected in this batch                  */
    uint32_t cand_overflow;
    uint32_t t2_sr;                 /* time2: shift register carried to the next batch     */
    uint32_t pad;
};

/* ---- geometry of the time2 pass ---------------------------------------------------------------
 * Five kernels per chain: k2t_count (one block per tile of T2_TILE_WORDS words: strobe count and last strobed bits of
 * the tile), the three-kernel scan t2scan_a/b/c over the tiles (their start ordinals and shift registers; the tiles
 * are its "lanes") and k2t_write (one block per tile again: the events into the ring).  In a tile, thread t loads
 * words 4t..4t+3 with 128-bit loads; for the events, "warp" w (T2_WARP consecutive threads) owns the tile's words
 * [w * T2_WARP * T2_WPT, +T2_WARP * T2_WPT) and handles them in T2_WPT rounds of T2_WARP consecutive words, lane l
 * taking the round's word l, so that a round's events are consecutive ordinals.  The CPU build uses tiny tiles and
 * "warps" so that its tests cross every boundary. */
#ifdef WMB_HOSTSIM
#define T2_THREADS 8
#define T2_WARP 4
#else
#define T2_THREADS 256
#define T2_WARP 32
#endif
#define T2_WPT 4                                /* words per thread (one 128-bit load each of sbits and dbits)     */
#define T2_TILE_WORDS (T2_THREADS * T2_WPT)
#define T2_WARPS (T2_THREADS / T2_WARP)
/* Staging holds one round of a warp, sized for the densest strobes the lock stencil allows: a strobe at m needs the
 * clock low at m-L-1 and high at m-L..m (lock_strobes), so strobes are at least L+2 >= 3 samples apart and a 32-sample
 * word holds at most 11 of them for every threshold 1..WMB_LOCK_MAX. */
#define T2_MIN_GAP 3
#define T2_MAX_PER_WORD 11
static_assert(T2_MAX_PER_WORD >= (32 + T2_MIN_GAP - 1) / T2_MIN_GAP, "time2 staging smaller than a dense round");
#define T2_STAGE (T2_WARP * T2_MAX_PER_WORD)

struct K2tParams {
    const uint32_t *dbits, *sbits;  /* 16-byte aligned                                      */
    const uint8_t *rssi;            /* index 0 = batch sample 0                             */
    int64_t  M;
    uint32_t lanes;                 /* tiles of T2_TILE_WORDS words, one block each         */
    uint32_t *cnt;                  /* [lanes] strobes per tile                             */
    uint32_t *tail;                 /* [lanes] last <=24 strobed bits, chronological        */
    uint32_t *tail_len;             /* [lanes]                                              */
    uint64_t *base;                 /* [lanes] ordinal of each tile's first event           */
    uint32_t *sr_start;             /* [lanes] shift register at the tile's first sample    */
    uint64_t *agg_cnt; uint32_t *agg_tail, *agg_len;   /* [scan tiles] scan scratch             */
    int64_t  m_base;
    uint64_t *ring; uint64_t ring_mask;
    StreamDev *sd;
    uint64_t *cand; uint32_t cand_cap;
    uint32_t ac_err;                /* access-code bit errors accepted (wmb_set_receiver)     */
};

WMB_HD uint32_t k2t_words(const K2tParams &p) { return (uint32_t)((p.M + 31) >> 5); }
WMB_HD uint32_t k2t_tiles(int64_t M) { return (uint32_t)(((M + 31) >> 5) + T2_TILE_WORDS - 1) / T2_TILE_WORDS; }

/* per tile: the strobe and data words of every tile word, and each word's first ordinal (relative to the tile's) and
 * shift register; the staged events of every warp's current round */
struct K2tSmem {
    uint32_t s[T2_TILE_WORDS], d[T2_TILE_WORDS];
    uint32_t ord[T2_TILE_WORDS], sr[T2_TILE_WORDS];
    uint64_t stage[T2_WARPS][T2_STAGE];
};

/* ---- device-wide exclusive scans over lanes -------------------------------------------------
 * Three small kernels: (A) every block of SCAN_BLOCK threads reduces a tile of SCAN_TILE lanes
 * (each thread a run of SCAN_ITEMS contiguous lanes), (B) one thread scans the tile aggregates,
 * (C) every block scans its tile again and writes the lanes' bases.  `part` is the block's
 * shared scratch (SCAN_BLOCK entries). */
#ifdef WMB_HOSTSIM                   /* tiny tiles so that the CPU tests cross tile boundaries */
#define SCAN_BLOCK 4
#define SCAN_ITEMS 2
#else
#define SCAN_BLOCK 256
#define SCAN_ITEMS 16
#endif
#define SCAN_TILE  (SCAN_BLOCK * SCAN_ITEMS)
#define SCAN_THREADS 1024            /* k3_offsets keeps the single-block variant */

WMB_HD uint32_t scan_per_thread(uint32_t n) { return (n + SCAN_THREADS - 1) / SCAN_THREADS; }
WMB_HD uint32_t scan_tiles(uint32_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }

struct CountScan {
    const uint32_t *cnt; uint64_t *base; uint32_t n;
    uint64_t *agg;                  /* [tiles] */
    uint64_t *total;                /* in: ordinal of the first item; out: += sum of cnt */
    const uint32_t *skip;           /* optional: nonzero -> leave everything untouched */
    uint32_t skip_invert;           /* ... zero -> leave everything untouched instead */
    uint32_t *clear;                /* optional: word zeroed by phase B */
    uint32_t from_zero;             /* ignore *total on input */
};

WMB_D void cscan_local(const CountScan &p, uint32_t tile, uint32_t tid, uint64_t *part)
{
    const uint32_t l0 = tile * SCAN_TILE + tid * SCAN_ITEMS;
    uint64_t s = 0;
#pragma unroll
    for (uint32_t i = 0; i < SCAN_ITEMS; i++) if (l0 + i < p.n) s += p.cnt[l0 + i];
    part[tid] = s;
}
WMB_D void cscan_a_finish(const CountScan &p, uint32_t tile, const uint64_t *part)
{
    uint64_t s = 0;
    for (uint32_t t = 0; t < SCAN_BLOCK; t++) s += part[t];
    p.agg[tile] = s;
}
WMB_D bool cscan_skipped(const CountScan &p) { return p.skip && ((*p.skip != 0) != (p.skip_invert != 0)); }

WMB_D void cscan_b(const CountScan &p)
{
    if (cscan_skipped(p)) return;
    uint64_t acc = p.from_zero ? 0 : *p.total;
    const uint32_t nt = scan_tiles(p.n);
    for (uint32_t t = 0; t < nt; t++) { const uint64_t c = p.agg[t]; p.agg[t] = acc; acc += c; }
    *p.total = acc;
    if (p.clear) *p.clear = 0;
}
WMB_D void cscan_c_block(const CountScan &p, uint32_t tile, uint64_t *part)
{
    uint64_t acc = p.agg[tile];
    for (uint32_t t = 0; t < SCAN_BLOCK; t++) { const uint64_t c = part[t]; part[t] = acc; acc += c; }
}
WMB_D void cscan_c_write(const CountScan &p, uint32_t tile, uint32_t tid, const uint64_t *part)
{
    if (cscan_skipped(p)) return;
    const uint32_t l0 = tile * SCAN_TILE + tid * SCAN_ITEMS;
    uint64_t acc = part[tid];
#pragma unroll
    for (uint32_t i = 0; i < SCAN_ITEMS; i++) if (l0 + i < p.n) { p.base[l0 + i] = acc; acc += p.cnt[l0 + i]; }
}

/* time2 variant: besides the strobe counts, the scan carries the shift register.  A lane contributes
 * its last <= 24 strobed bits (tail, len); appending `len` newer bits shifts the older ones up, which
 * is associative, so (register, tail) pairs fold like sums. */
struct T2Fold { uint64_t cnt; uint32_t tail, len; };

template <class CH>
WMB_D void t2_append(T2Fold &a, uint64_t cnt, uint32_t tail, uint32_t len)
{
    constexpr uint32_t NB = (CH::ID == 0) ? 16 : 24;
    a.cnt += cnt;
    a.tail = (uint32_t)((((uint64_t)a.tail << len) | tail) & CH::CODE_MASK);
    a.len = (a.len + len > NB) ? NB : a.len + len;
}

template <class CH>
WMB_D void t2scan_local(const K2tParams &p, uint32_t tile, uint32_t tid, T2Fold *part)
{
    const uint32_t l0 = tile * SCAN_TILE + tid * SCAN_ITEMS;
    T2Fold f = { 0, 0, 0 };
#pragma unroll
    for (uint32_t i = 0; i < SCAN_ITEMS; i++) if (l0 + i < p.lanes) t2_append<CH>(f, p.cnt[l0 + i], p.tail[l0 + i], p.tail_len[l0 + i]);
    part[tid] = f;
}
template <class CH>
WMB_D void t2scan_a_finish(const K2tParams &p, uint32_t tile, const T2Fold *part)
{
    T2Fold f = { 0, 0, 0 };
    for (uint32_t t = 0; t < SCAN_BLOCK; t++) t2_append<CH>(f, part[t].cnt, part[t].tail, part[t].len);
    p.agg_cnt[tile] = f.cnt; p.agg_tail[tile] = f.tail; p.agg_len[tile] = f.len;
}
template <class CH>
WMB_D void t2scan_b(const K2tParams &p)
{
    uint64_t acc = p.sd->total;
    uint64_t sr = p.sd->t2_sr;
    const uint32_t nt = scan_tiles(p.lanes);
    for (uint32_t t = 0; t < nt; t++) {
        const uint64_t c = p.agg_cnt[t];
        const uint32_t tl = p.agg_tail[t], ll = p.agg_len[t];
        p.agg_cnt[t] = acc; p.agg_tail[t] = (uint32_t)sr;            /* exclusive prefixes */
        acc += c;
        sr = ((sr << ll) | tl) & CH::CODE_MASK;
    }
    p.sd->total = acc;
    p.sd->t2_sr = (uint32_t)sr;
}
template <class CH>
WMB_D void t2scan_c_block(const K2tParams &p, uint32_t tile, T2Fold *part)
{
    uint64_t acc = p.agg_cnt[tile];
    uint64_t sr = p.agg_tail[tile];
    for (uint32_t t = 0; t < SCAN_BLOCK; t++) {
        const T2Fold f = part[t];
        part[t].cnt = acc; part[t].tail = (uint32_t)sr;               /* exclusive prefixes */
        acc += f.cnt;
        sr = ((sr << f.len) | f.tail) & CH::CODE_MASK;
    }
}
template <class CH>
WMB_D void t2scan_c_write(const K2tParams &p, uint32_t tile, uint32_t tid, const T2Fold *part)
{
    const uint32_t l0 = tile * SCAN_TILE + tid * SCAN_ITEMS;
    uint64_t acc = part[tid].cnt;
    uint64_t sr = part[tid].tail;
#pragma unroll
    for (uint32_t i = 0; i < SCAN_ITEMS; i++) {
        if (l0 + i >= p.lanes) break;
        p.base[l0 + i] = acc; p.sr_start[l0 + i] = (uint32_t)sr;
        acc += p.cnt[l0 + i];
        sr = ((sr << p.tail_len[l0 + i]) | p.tail[l0 + i]) & CH::CODE_MASK;
    }
}


template <class CH>
WMB_D T2Fold t2_fold(T2Fold a, const T2Fold &b) { t2_append<CH>(a, b.cnt, b.tail, b.len); return a; }

/* one word: its strobed data bits, oldest first (the newest in bit 0) */
template <class CH>
WMB_D T2Fold t2_word(uint32_t s, uint32_t d)
{
    constexpr uint32_t NB = (CH::ID == 0) ? 16 : 24;
    T2Fold f = { (uint64_t)wmb_popc(s), 0u, 0u };
    while (s) {
        const int i = wmb_ffs(s) - 1;
        s &= s - 1;
        f.tail = (f.tail << 1) | ((d >> i) & 1u);
    }
    f.tail &= CH::CODE_MASK;
    f.len = f.cnt > NB ? NB : (uint32_t)f.cnt;
    return f;
}

/* k2t_count / k2t_write, phase 1: thread `tid` loads its four words of the tile (zero past the batch), keeps them in
 * `sm` when given, and returns their fold */
template <class CH>
WMB_D T2Fold k2t_load(const K2tParams &p, uint32_t tile, uint32_t tid, K2tSmem *sm)
{
    const uint32_t nw = k2t_words(p), w = tile * T2_TILE_WORDS + tid * T2_WPT;
    uint32_t s4[T2_WPT], d4[T2_WPT];
    if (w + T2_WPT <= nw) {
        const u32x4 sv = *(const u32x4 *)(p.sbits + w), dv = *(const u32x4 *)(p.dbits + w);
        s4[0] = sv.x; s4[1] = sv.y; s4[2] = sv.z; s4[3] = sv.w;
        d4[0] = dv.x; d4[1] = dv.y; d4[2] = dv.z; d4[3] = dv.w;
    } else {
#pragma unroll
        for (int q = 0; q < T2_WPT; q++) { s4[q] = (w + q < nw) ? p.sbits[w + q] : 0u; d4[q] = (w + q < nw) ? p.dbits[w + q] : 0u; }
    }
    T2Fold f = { 0, 0, 0 };
#pragma unroll
    for (int q = 0; q < T2_WPT; q++) {
        f = t2_fold<CH>(f, t2_word<CH>(s4[q], d4[q]));
        if (sm) { sm->s[tid * T2_WPT + q] = s4[q]; sm->d[tid * T2_WPT + q] = d4[q]; }
    }
    return f;
}

/* k2t_count, last phase: the tile's aggregate (the scan's inclusive total from the identity) */
WMB_D void k2t_count_store(const K2tParams &p, uint32_t tile, const T2Fold &total)
{
    p.cnt[tile] = (uint32_t)total.cnt; p.tail[tile] = total.tail; p.tail_len[tile] = total.len;
}

/* k2t_write: the carry into the tile's scan -- ordinals relative to the tile's first event, and its start register */
template <class CH>
WMB_D T2Fold k2t_carry(const K2tParams &p, uint32_t tile)
{
    constexpr uint32_t NB = (CH::ID == 0) ? 16 : 24;
    const T2Fold c = { 0, p.sr_start[tile], NB };
    return c;
}
/* k2t_write, after the scan: thread `tid` spreads its exclusive prefix over its four words */
template <class CH>
WMB_D void k2t_spread(uint32_t tid, T2Fold acc, K2tSmem &sm)
{
#pragma unroll
    for (int q = 0; q < T2_WPT; q++) {
        const uint32_t w = tid * T2_WPT + q;
        sm.ord[w] = (uint32_t)acc.cnt; sm.sr[w] = acc.tail;
        acc = t2_fold<CH>(acc, t2_word<CH>(sm.s[w], sm.d[w]));
    }
}

/* k2t_write, round r: lane l of warp w produces the events of the round's word l into the warp's staging (at their
 * ordinal's offset from the round's first), and appends its access-code matches to the candidate list */
WMB_HD uint32_t k2t_round_word(uint32_t tid, uint32_t r)
{
    return (tid / T2_WARP) * (T2_WARP * T2_WPT) + r * T2_WARP + tid % T2_WARP;
}
template <class CH>
WMB_D void k2t_emit(const K2tParams &p, uint32_t tile, uint32_t tid, uint32_t r, K2tSmem &sm)
{
    const uint32_t w = k2t_round_word(tid, r);
    uint32_t s = sm.s[w];
    if (!s) return;
    const uint32_t d = sm.d[w];
    uint64_t *stage = sm.stage[tid / T2_WARP] + (sm.ord[w] - sm.ord[k2t_round_word(tid - tid % T2_WARP, r)]);
    uint64_t ord = p.base[tile] + sm.ord[w];
    uint32_t sr = sm.sr[w];
    const int64_t word = (int64_t)tile * T2_TILE_WORDS + w;
    const u32x4 *r4 = (const u32x4 *)(p.rssi + word * 32);           /* 32-byte aligned */
    const u32x4 rs[2] = { r4[0], r4[1] };
    while (s) {
        const int i = wmb_ffs(s) - 1;
        s &= s - 1;
        const uint32_t bit = (d >> i) & 1u;
        sr = ((sr << 1) | bit) & CH::CODE_MASK;                      /* rtl_wmbus.c:820 */
        const uint32_t sync = ac_match<CH>(sr, p.ac_err);            /* rtl_wmbus.c:822 */
        const u32x4 rq = rs[i >> 4];
        const uint32_t rw = ((i >> 2) & 3) == 0 ? rq.x : ((i >> 2) & 3) == 1 ? rq.y : ((i >> 2) & 3) == 2 ? rq.z : rq.w;
        const uint32_t rssi = (rw >> (8 * (i & 3))) & 0xFFu;
        *stage++ = ((uint64_t)(p.m_base + word * 32 + i) << 24) | ((uint64_t)rssi << 16) | (sync << 1) | bit;
        if (sync) {
#ifdef WMB_HOSTSIM
            const uint32_t slot = p.sd->n_cand++;
#else
            const uint32_t slot = atomicAdd(&p.sd->n_cand, 1u);
#endif
            if (slot < p.cand_cap) p.cand[slot] = ord;
            else p.sd->cand_overflow = 1;
        }
        ord++;
    }
}
/* k2t_write, round r after the warp's emits: its lanes copy the staged events to the ring in ordinal order, so that a
 * warp's stores cover consecutive slots (split only where the ring wraps) */
WMB_D void k2t_flush(const K2tParams &p, uint32_t tile, uint32_t tid, uint32_t r, const K2tSmem &sm)
{
    const uint32_t l = tid % T2_WARP, first = k2t_round_word(tid - l, r), last = first + T2_WARP - 1;
    const uint32_t n = sm.ord[last] + (uint32_t)wmb_popc(sm.s[last]) - sm.ord[first];
    const uint64_t ord0 = p.base[tile] + sm.ord[first];
    const uint64_t *stage = sm.stage[tid / T2_WARP];
    for (uint32_t i = l; i < n; i += T2_WARP) p.ring[(ord0 + i) & p.ring_mask] = stage[i];
}

/* ------------------------------------------------------------------------------------- */
/* K2m: run-length lanes                                                                 */
/* ------------------------------------------------------------------------------------- */

struct K2mParams {
    const uint32_t *dbits;      /* word index 0 = batch sample 0; history at negative indices */
    const uint8_t *rssi;
    int64_t  M, hist;
    uint32_t C, W, lanes;
    uint32_t cap;               /* per-lane event capacity                                    */
    uint32_t *ev;               /* [lanes * cap] lane-local events                            */
    uint32_t *cnt;              /* [lanes]                                                    */
    RlState *st_start, *st_end;
    const RlState *carry;
    uint32_t *rerun;
    uint32_t *errors;           /* bit0 event overflow, bit1 run-length tracker out of range  */
    uint32_t *lane_err;         /* [lanes] the same bits per lane: a speculative lane that started from the wrong state may
                                   overflow its buffer or leave the tracker's range without the stream doing so -- only
                                   what a lane's LAST run (the verified one) reports counts, and K2c collects it        */
    uint32_t mode;
    const uint32_t *run_if;     /* optional: the whole pass happens only if this word is nonzero (T1/C1 fallback
                                   from the two-phase path, decided on the device)                */
    uint32_t ac_err;            /* access-code bit errors accepted (wmb_set_receiver)         */
};

struct K2Out { uint32_t *ev; uint32_t cap; uint32_t n; uint32_t overflow; };

WMB_D void k2_emit(K2Out &o, bool live, uint32_t off, uint32_t rssi, uint32_t rst, uint32_t sync, uint32_t bit)
{
    if (!live) return;
    if (o.n < o.cap) o.ev[o.n] = EV_LOCAL(off, rssi, rst, sync, bit);
    else o.overflow = 1;
    o.n++;
}

/* an edge of the deglitched stream: decide between reset and bit emission */
template <class CH>
WMB_D bool k2m_edge(const K2mParams &p, RlState &s, uint32_t st, int64_t m, uint32_t off, bool live,
                    K2Out &o, uint32_t &err)
{
    const uint32_t level = s.flags & 1u;
    bool reset = false;
    int n = 0;
    if (CH::ID == 0) {                                       /* rtl_wmbus.c:742-796 */
        if (s.run < 5) reset = true;
        else {
            int rl = s.run * 256;
            const int half = s.a / 2;
            if (rl <= half) reset = true;
            else if (s.a <= 0) { reset = true; err |= 2u; }  /* the reference would spin here */
            else {
                const uint32_t rssi = 0u;                    /* filled in by k2c_compact */
                while (rl > half) {
                    rl -= s.a;
                    s.sr = ((s.sr << 1) | level) & CH::CODE_MASK;
                    if (n < K2_EDGE_EMIT_CAP) {
                        k2_emit(o, live, off, rssi, (s.flags >> 1) & 1u, ac_match<CH>(s.sr, p.ac_err), level);
                        s.flags &= ~2u;
                    }
                    n++;
                }
                s.b += rl;
                s.a += (rl + s.b / 16) / (32 * n);
            }
        }
        if (reset) { s.a = 8 * 256; s.b = 0; }
    } else {                                                 /* rtl_wmbus.c:655-698 */
        const int spb = (s.a + s.b) / 2;
        const int half = spb / 2;
        const int run = s.run;
        if (spb <= 12 || spb >= 36) reset = true;
        else if (run <= half) reset = true;
        else {
            int rl = run;
            const uint32_t rssi = 0u;                        /* filled in by k2c_compact */
            while (rl > half) {
                rl -= spb;
                s.sr = ((s.sr << 1) | level) & CH::CODE_MASK;
                if (n < K2_EDGE_EMIT_CAP) {
                    k2_emit(o, live, off, rssi, (s.flags >> 1) & 1u, ac_match<CH>(s.sr, p.ac_err), level);
                    s.flags &= ~2u;
                }
                n++;
            }
            if (level) s.b = run / n; else s.a = run / n;
        }
        if (reset) { s.a = 24; s.b = 24; }
    }
    if (reset) {                                             /* runlength_algorithm_reset_* */
        s.raw = 0; s.sr = 0;
        s.flags = 2u;                                        /* decoder reset: frames are cut here */
    }
    s.flags = (s.flags & ~1u) | st;
    s.run = 1;
    return reset;
}

/* Deglitched level of 32 consecutive samples at once.  H holds raw bits in time order: bit K + i is
 * sample i of the current word, bits 0..K-1 are the K samples before it (K = 5 for T1/C1, 3 for S1);
 * bits that precede the last reset are zero (the reference clears its history on reset, :717-726). */
template <class CH>
WMB_D uint32_t k2m_deglitch_word(uint64_t H)
{
    if (CH::ID == 0) {
        /* at least 3 of the 6 most recent bits (deglitch_filter_t1_c1, rtl_wmbus.c:126-144), as a
         * bit-sliced addition: a+b+c = 2*c1 + s1, d+e+f = 2*c2 + s2 */
        const uint64_t a = H >> 5, bb = H >> 4, c = H >> 3, d = H >> 2, e = H >> 1, f = H;
        const uint64_t s1 = a ^ bb ^ c, c1 = (a & bb) | (c & (a ^ bb));
        const uint64_t s2 = d ^ e ^ f, c2 = (d & e) | (f & (d ^ e));
        return (uint32_t)((c1 & c2) | ((c1 ^ c2) & (s1 | s2)));
    } else {
        /* newest bit, or at least two of the three before it (deglitch_filter_s1, rtl_wmbus.c:149-154) */
        const uint64_t b0 = H >> 3, b1 = H >> 2, b2 = H >> 1, b3 = H;
        return (uint32_t)(b0 | (b1 & b2) | (b1 & b3) | (b2 & b3));
    }
}

/* the reference keeps its raw history with the newest bit in bit 0; the lanes keep it in time order.
 * Only the K most recent bits matter for what follows, so the state carries exactly those. */
template <class CH>
WMB_D uint64_t k2m_hist_from_raw(uint32_t raw)
{
    constexpr int K = (CH::ID == 0) ? 5 : 3;
    uint64_t h = 0;
#pragma unroll
    for (int j = 0; j < K; j++) h |= (uint64_t)((raw >> j) & 1u) << (K - 1 - j);
    return h;
}
template <class CH>
WMB_D uint32_t k2m_raw_from_hist(uint64_t h)
{
    constexpr int K = (CH::ID == 0) ? 5 : 3;
    uint32_t raw = 0;
#pragma unroll
    for (int j = 0; j < K; j++) raw |= (uint32_t)((h >> (K - 1 - j)) & 1u) << j;
    return raw;
}

/* Run-length lane, edge driven: the deglitched level of a whole 32-sample word comes from a few
 * bitwise operations, the lane then jumps from edge to edge (ffs) instead of stepping through samples.
 * (It replaces a version that stepped through every sample.) */
template <class CH>
WMB_D void k2m_lane(const K2mParams &p, uint32_t lane)
{
    if (lane >= p.lanes) return;
    if (p.run_if && !*p.run_if) return;
    constexpr int K = (CH::ID == 0) ? 5 : 3;
    const int64_t s0 = (int64_t)lane * p.C;
    const int64_t e0 = (s0 + p.C < p.M) ? s0 + p.C : p.M;
    RlState s;
    int64_t m;
    if (p.mode == 0) {
        if (lane == 0) { s = *p.carry; m = 0; }
        else {
            rl_state_init(s, CH::ID);
            m = s0 - (int64_t)p.W;
            if (m < -p.hist) m = -p.hist;
        }
    } else {
        if (lane == 0 || !p.rerun[lane]) return;
        s = p.st_end[lane - 1];
        m = s0;
    }
    K2Out o = { p.ev + (size_t)lane * p.cap, p.cap, 0, 0 };
    uint32_t err = 0;
    bool saved_start = false;
    uint64_t H = k2m_hist_from_raw<CH>(s.raw);                 /* K history bits */
    /* words are fetched eight at a time (one 32-byte sector per lane) and the next eight are requested
     * before the current ones are walked: with one warp per scheduler a dependent load per word would
     * expose the full DRAM latency 4600 times per lane */
    uint32_t wcur[8], wnxt[8];
    {
        const u32x4 *src = (const u32x4 *)(p.dbits + (m >> 5));
        const u32x4 a = src[0], c = src[1];
        wcur[0] = a.x; wcur[1] = a.y; wcur[2] = a.z; wcur[3] = a.w; wcur[4] = c.x; wcur[5] = c.y; wcur[6] = c.z; wcur[7] = c.w;
    }
    while (m < e0) {
        {
            const u32x4 *src = (const u32x4 *)(p.dbits + (m >> 5) + 8);     /* slack behind M covers the over-read */
            const u32x4 a = src[0], c = src[1];
            wnxt[0] = a.x; wnxt[1] = a.y; wnxt[2] = a.z; wnxt[3] = a.w; wnxt[4] = c.x; wnxt[5] = c.y; wnxt[6] = c.z; wnxt[7] = c.w;
        }
#pragma unroll
        for (int q = 0; q < 8; q++) {
            if (m >= e0) break;
            if (m == s0 && !saved_start) {
                s.raw = k2m_raw_from_hist<CH>(H);
                p.st_start[lane] = s;
                saved_start = true;
            }
            const int n = (e0 - m >= 32) ? 32 : (int)(e0 - m);
            const uint32_t valid = (n == 32) ? 0xFFFFFFFFu : ((1u << n) - 1u);
            const uint32_t word = wcur[q] & valid;
            const bool live = m >= s0;
            H = (H & ((1ull << K) - 1)) | ((uint64_t)word << K);
            int pos = 0;                                       /* next unprocessed in-word position */
            while (pos < n) {
                const uint32_t D = k2m_deglitch_word<CH>(H);
                const uint32_t lvl = (s.flags & 1u) ? 0xFFFFFFFFu : 0u;
                const uint32_t x = (D ^ lvl) & (0xFFFFFFFFu << pos) & valid;
                if (!x) { s.run += n - pos; break; }
                const int e = wmb_ffs(x) - 1;
                s.run += e - pos;                              /* samples that kept the level */
                const bool reset = k2m_edge<CH>(p, s, (D >> e) & 1u, m + e, (uint32_t)(m + e - s0), live, o, err);
                if (reset) H &= ~((1ull << (K + e + 1)) - 1);  /* forget every bit up to and including e */
                pos = e + 1;
            }
            m += n;
            H >>= n;                                           /* the newest K bits become the history */
        }
#pragma unroll
        for (int q = 0; q < 8; q++) wcur[q] = wnxt[q];
    }
    s.raw = k2m_raw_from_hist<CH>(H);
    if (!saved_start) p.st_start[lane] = s;
    p.st_end[lane] = s;
    p.cnt[lane] = o.n < o.cap ? o.n : o.cap;
    if (o.overflow) err |= 1u;
    if (p.lane_err) p.lane_err[lane] = err;
    else if (err) {
#ifdef WMB_HOSTSIM
        *p.errors |= err;
#else
        atomicOr(p.errors, err);
#endif
    }
}

WMB_D void k2m_verify_lane(const K2mParams &p, uint32_t lane, uint32_t *n_fail)
{
    if (lane >= p.lanes) return;
    if (p.run_if && !*p.run_if) return;
    uint32_t bad = 0;
    if (lane > 0) {
        const RlState &a = p.st_start[lane], &b = p.st_end[lane - 1];
        if (!(a.run == b.run && a.a == b.a && a.b == b.b && a.flags == b.flags && a.raw == b.raw && a.sr == b.sr)) bad = 1;
    }
    p.rerun[lane] = bad;
    if (bad) {
#ifdef WMB_HOSTSIM
        (*n_fail)++;
#else
        atomicAdd(n_fail, 1u);
#endif
    }
}

/* ------------------------------------------------------------------------------------- */
/* K2p: two-phase run-length bit sync for the T1/C1 chain                                */
/*                                                                                       */
/* The reference's run-length algorithm (rtl_wmbus.c:729-803) mixes two time scales: a    */
/* per-sample deglitch/edge detector whose only feedback is "runs shorter than 5 samples  */
/* reset everything", and a per-run PI loop that turns run lengths into bits.  Phase 1    */
/* keeps the per-sample part (a tiny state: 6 raw bits, level, run length, a pending-     */
/* reset flag) and emits one RECORD per run of >= 5 samples; phase 2 walks the records.   */
/* A record that follows a reset starts phase 2 from a known state, so phase 2 is exactly */
/* segment-parallel.  The one coupling phase 1 cannot see is the reference's second reset */
/* rule (run*256 <= bit_length/2 with run >= 5, :756-762), which needs a bit_length 25 %   */
/* above nominal; phase 2 detects it and the batch falls back to the exact monolithic     */
/* lanes (k2m_lane).                                                                      */
/* ------------------------------------------------------------------------------------- */

struct P1State { uint32_t raw, level, pend; int32_t run; };

struct K2p1Params {
    const uint32_t *dbits;
    int64_t  M, hist;
    uint32_t C, W, lanes;       /* multiples of 32 */
    uint32_t cap;               /* records per lane */
    uint64_t *rec;              /* [lanes * cap] lane-local records: run<<32 | off<<2 | level<<1 | rst */
    uint32_t *cnt;              /* [lanes] */
    P1State *st_start, *st_end;
    const RlState *carry;
    uint32_t *rerun;
    uint32_t mode;
};

WMB_D void k2p1_lane(const K2p1Params &p, uint32_t lane)
{
    if (lane >= p.lanes) return;
    const int64_t s0 = (int64_t)lane * p.C;
    const int64_t e0 = (s0 + p.C < p.M) ? s0 + p.C : p.M;
    uint32_t raw, level, pend;
    int32_t run;
    int64_t m;
    if (p.mode == 0) {
        if (lane == 0) {
            const RlState c = *p.carry;
            raw = c.raw; level = c.flags & 1u; pend = (c.flags >> 1) & 1u; run = c.run; m = 0;
        } else {
            raw = 0; level = 0; pend = 0; run = 0;
            m = s0 - (int64_t)p.W;
            if (m < -p.hist) m = -p.hist;
        }
    } else {
        if (lane == 0 || !p.rerun[lane]) return;
        const P1State c = p.st_end[lane - 1];
        raw = c.raw; level = c.level; pend = c.pend; run = c.run; m = s0;
    }
    uint64_t *rec = p.rec + (size_t)lane * p.cap;
    uint32_t n_rec = 0;
    bool saved_start = false;
    /* edge driven like k2m_lane: the deglitched level of a whole word comes from a few bitwise
     * operations (recomputed only after a reset, which clears the raw history), then the lane jumps
     * from edge to edge.  The state keeps the K = 5 raw bits that can still matter. */
    constexpr int K = 5;
    uint64_t H = k2m_hist_from_raw<ChainT1C1>(raw);
    uint32_t wnext = (m < e0) ? p.dbits[m >> 5] : 0u;
    while (m < e0) {
        if (m == s0 && !saved_start) {
            P1State st = { k2m_raw_from_hist<ChainT1C1>(H), level, pend, run };
            p.st_start[lane] = st; saved_start = true;
        }
        const int n = (e0 - m >= 32) ? 32 : (int)(e0 - m);
        const uint32_t valid = (n == 32) ? 0xFFFFFFFFu : ((1u << n) - 1u);
        const uint32_t word = wnext & valid;
        if (m + 32 < e0) wnext = p.dbits[(m >> 5) + 1];              /* request the next word early */
        const bool live = m >= s0;
        H = (H & ((1ull << K) - 1)) | ((uint64_t)word << K);
        uint32_t D = k2m_deglitch_word<ChainT1C1>(H);
        int pos = 0;
        while (pos < n) {
            const uint32_t x = (D ^ (level ? 0xFFFFFFFFu : 0u)) & (0xFFFFFFFFu << pos) & valid;
            if (!x) { run += n - pos; break; }
            const int e = wmb_ffs(x) - 1;
            run += e - pos;                                          /* samples that kept the level */
            const uint32_t st = (D >> e) & 1u;
            if (run < 5) {                                           /* :742-748: forget every bit up to and including e */
                H &= ~((1ull << (K + e + 1)) - 1);
                D = k2m_deglitch_word<ChainT1C1>(H);
                pend = 1;
            } else {
                if (live && n_rec < p.cap)
                    rec[n_rec] = ((uint64_t)(uint32_t)run << 32) | ((uint64_t)(uint32_t)(m + e - s0) << 2) | (level << 1) | pend;
                if (live) n_rec++;
                pend = 0;
            }
            level = st; run = 1;
            pos = e + 1;
        }
        m += n;
        H >>= n;                                                     /* the newest K bits become the history */
    }
    raw = k2m_raw_from_hist<ChainT1C1>(H);
    P1State st = { raw, level, pend, run };
    if (!saved_start) p.st_start[lane] = st;
    p.st_end[lane] = st;
    p.cnt[lane] = n_rec < p.cap ? n_rec : p.cap;     /* cap = C/5 + 2 cannot overflow: runs are >= 5 samples */
}

WMB_D void k2p1_verify_lane(const K2p1Params &p, uint32_t lane, uint32_t *n_fail)
{
    if (lane >= p.lanes) return;
    uint32_t bad = 0;
    if (lane > 0) {
        const P1State &a = p.st_start[lane], &b = p.st_end[lane - 1];
        if (!(a.raw == b.raw && a.level == b.level && a.pend == b.pend && a.run == b.run)) bad = 1;
    }
    p.rerun[lane] = bad;
    if (bad) {
#ifdef WMB_HOSTSIM
        (*n_fail)++;
#else
        atomicAdd(n_fail, 1u);
#endif
    }
}

/* records -> one global list per batch */
struct K2pDev {                 /* device bookkeeping of the two-phase path */
    uint64_t n_rec;             /* records in this batch                                   */
    uint32_t fallback;          /* phase 2 met the second reset rule: redo with k2m_lane   */
    uint32_t errors;
};

struct K2pcParams {
    const uint64_t *rec; const uint32_t *cnt; uint64_t *base;
    uint32_t lanes, cap, C;
    uint32_t *rec_m, *rec_v;    /* out: batch-relative edge sample ; run<<2 | level<<1 | rst */
    uint64_t *agg;
    K2pDev *pd;
};

WMB_D void k2pc_compact(const K2pcParams &p, uint32_t lane, int tid, int nthr)
{
    if (lane >= p.lanes) return;
    const uint32_t n = p.cnt[lane];
    const uint64_t base = p.base[lane];
    const uint64_t *src = p.rec + (size_t)lane * p.cap;
    for (uint32_t i = tid; i < n; i += nthr) {
        const uint64_t r = src[i];
        uint64_t run = r >> 32;
        if (run > 0x3FFFFFFFu) run = 0x3FFFFFFFu;
        p.rec_m[base + i] = (uint32_t)((uint64_t)lane * p.C + ((r >> 2) & 0x3FFFFFFFu));
        p.rec_v[base + i] = (uint32_t)(run << 2) | (uint32_t)(r & 3u);
    }
}

/* phase 2 */
struct K2p2Params {
    const uint32_t *rec_m, *rec_v;
    uint16_t *rec_n;            /* [records] bits emitted per record (pass A -> pass B)     */
    K2pDev *pd;
    uint32_t R;                 /* records per lane (nominal)                              */
    uint32_t lanes;
    uint32_t *cnt;              /* [lanes] events per lane                                 */
    uint64_t *base;             /* [lanes]                                                 */
    const uint8_t *rssi;
    int64_t  m_base;
    uint64_t *ring; uint64_t ring_mask;
    StreamDev *sd;
    uint64_t *cand; uint32_t cand_cap;
    const RlState *carry;       /* exact state at batch start                               */
    RlState *p2_out;            /* out: a/b/sr after the last record, run = 1 marks it valid */
    uint64_t *agg;
    uint32_t ac_err;            /* access-code bit errors accepted (wmb_set_receiver)       */
};

#define K2P2_BLK 8                   /* records fetched together (memory-level parallelism) */
#define K2P2W_THREADS 128            /* write pass: one block per lane of records */
#define K2P2W_ITEMS 4                /* consecutive records per thread (K2P2W_THREADS * K2P2W_ITEMS >= R) */

/* C integer division (truncation toward zero) by 2^s and by a small positive n */
WMB_D int wmb_div_pow2(int x, int s) { return (x + ((x >> 31) & ((1 << s) - 1))) >> s; }
/* x / n for 1 <= n <= 8 and |x| < 2^29 without a divide or a jump table: |x| * ceil(2^35 / n) >> 35
 * is exact as long as |x| < 2^35 / n */
WMB_D int wmb_div_small(int x, int n)
{
    static const uint64_t magic[9] = { 0, 1ull << 35, 1ull << 34, 11453246123ull, 1ull << 33, 6871947674ull, 5726623062ull,
                                4908534053ull, 1ull << 32 };
    const uint32_t ax = (uint32_t)(x < 0 ? -x : x);
    const int q = (int)(((uint64_t)ax * magic[n]) >> 35);
    return x < 0 ? -q : q;
}

/* pass A (serial in the PI recurrence, nothing else): bits per record -> rec_n.  A lane owns the
 * records from the first reset in its range up to the first reset of a later range, so a telegram
 * (which has no reset inside) is one dependent chain; the step is therefore written for latency:
 * no loop and no jump table on the way from one bit-length estimate to the next.
 * Only rec_v is read; the next block of records is requested while the current one is processed. */
WMB_D void k2p2_count(const K2p2Params &p, uint32_t lane)
{
    if (lane >= p.lanes) return;
    const uint32_t N = (uint32_t)p.pd->n_rec;                        /* < 2^32: at most one record per five samples */
    const uint64_t r0w = (uint64_t)lane * p.R;
    if (r0w >= N) return;
    const uint32_t r0 = (uint32_t)r0w, r1 = (N - r0 > p.R) ? r0 + p.R : N;
    uint32_t i = r0;
    if (lane != 0) {                                                 /* the lane's first record: the first one in its range that follows a reset */
        while (i < r1 && !(p.rec_v[i] & 1u)) i++;
        if (i >= r1) return;
    }
    int32_t a = 8 * 256, b = 0;
    if (lane == 0) { const RlState c = *p.carry; a = c.a; b = c.b; }
    bool stop = false, ran_off_end = false;
    uint32_t v[K2P2_BLK], vn[K2P2_BLK];
#pragma unroll
    for (int j = 0; j < K2P2_BLK; j++) v[j] = (i + j < N) ? p.rec_v[i + j] : 1u;
    while (!stop) {
#pragma unroll
        for (int j = 0; j < K2P2_BLK; j++) vn[j] = (i + K2P2_BLK + j < N) ? p.rec_v[i + K2P2_BLK + j] : 1u;
#pragma unroll
        for (int j = 0; j < K2P2_BLK; j++) {
            if (stop) continue;
            const uint32_t idx = i + j;
            if (idx >= N) { stop = true; ran_off_end = true; continue; }
            const uint32_t vv = v[j];
            if (vv & 1u) {
                if (idx >= r1) { stop = true; continue; }            /* next lane's segment */
                a = 8 * 256; b = 0;                                  /* runlength_algorithm_reset_t1_c1 */
            }
            const int32_t rl0 = (int32_t)((vv >> 2) << 8);
            const int32_t half = a / 2;
            if (rl0 <= half || a <= 0) {                             /* rtl_wmbus.c:756-762 (or a spin) */
                p.pd->fallback = 1;
                stop = true; continue;
            }
            /* n = number of bit periods in the run (:765-779): the smallest n with rl0 - n*a <= half.  Telegram runs
             * are 1-4 bits long: compare against all of half + k*a at once (independent compares: the pass is bound by
             * the latency of this per-record chain -- a reciprocal-estimate quotient measured 15 % slower) and keep
             * the integer division for the rare long run. */
            int32_t n, rl = rl0;
            if (rl - half <= 8 * a) {
                n = 1;
                int32_t th = half;
#pragma unroll
                for (int k = 1; k < 8; k++) { th += a; n += (rl > th) ? 1 : 0; }
                rl -= n * a;
                b += rl;                                             /* :792 */
                a += wmb_div_small(wmb_div_pow2(rl + wmb_div_pow2(b, 4), 5), n);   /* :796: x/(32 n) == (x/32)/n */
            } else {
                n = (rl - half + a - 1) / a; rl -= n * a;
                b += rl;
                a += wmb_div_pow2(rl + wmb_div_pow2(b, 4), 5) / n;
            }
            p.rec_n[idx] = (uint16_t)(n < K2_EDGE_EMIT_CAP ? n : K2_EDGE_EMIT_CAP);
        }
        i += K2P2_BLK;
#pragma unroll
        for (int j = 0; j < K2P2_BLK; j++) v[j] = vn[j];
    }
    if (ran_off_end) { p.p2_out->a = a; p.p2_out->b = b; }           /* exactly one lane sees the last record */
}

/* pass B: with the bit counts known nothing is serial any more.  One block per lane of R records,
 * K2P2W_ITEMS consecutive records per thread: (a) per-thread bit counts, (b) their exclusive scan,
 * (c) every thread rebuilds the 16-bit shift register in front of its first record from the
 * preceding records (at most 16 of them, or the carried register at the start of the batch) and
 * writes its records' events with the access-code test. */
WMB_D void k2p2w_a(const K2p2Params &p, uint32_t lane, uint32_t tid, uint32_t *part)
{
    uint32_t s = 0;
    if (!p.pd->fallback) {
        const uint64_t N = p.pd->n_rec;
        const uint64_t r0 = (uint64_t)lane * p.R, r1 = (r0 + p.R < N) ? r0 + p.R : N;
        const uint64_t i0 = r0 + (uint64_t)tid * K2P2W_ITEMS;
#pragma unroll
        for (int j = 0; j < K2P2W_ITEMS; j++) if (i0 + j < r1) s += p.rec_n[i0 + j];
    }
    part[tid] = s;
}

/* events per lane of records = sum of part[] after k2p2w_a */
WMB_D void k2p2_sum_finish(const K2p2Params &p, uint32_t lane, const uint32_t *part)
{
    uint32_t n_ev = 0;
    for (uint32_t t = 0; t < K2P2W_THREADS; t++) n_ev += part[t];
    p.cnt[lane] = n_ev;
}

/* exclusive scan of part[0 .. K2P2W_THREADS) */
#ifdef WMB_HOSTSIM
static inline void k2p2w_b(uint32_t *part, uint32_t)
{
    uint32_t acc = 0;
    for (uint32_t t = 0; t < K2P2W_THREADS; t++) { const uint32_t c = part[t]; part[t] = acc; acc += c; }
}
#else
WMB_D void k2p2w_b(uint32_t *part, uint32_t tid)
{
    if (tid >= 32) return;
    constexpr int PER = K2P2W_THREADS / 32;
    uint32_t loc[PER], tot = 0;
#pragma unroll
    for (int k = 0; k < PER; k++) { loc[k] = tot; tot += part[tid * PER + k]; }
    uint32_t inc = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)tid >= d) inc += o; }
    const uint32_t excl = inc - tot;
#pragma unroll
    for (int k = 0; k < PER; k++) part[tid * PER + k] = excl + loc[k];
}
#endif

WMB_D void k2p2w_c(const K2p2Params &p, uint32_t lane, uint32_t tid, const uint32_t *part)
{
    if (p.pd->fallback) return;
    const uint64_t N = p.pd->n_rec;
    const uint64_t r0 = (uint64_t)lane * p.R, r1 = (r0 + p.R < N) ? r0 + p.R : N;
    const uint64_t i0 = r0 + (uint64_t)tid * K2P2W_ITEMS;
    if (i0 >= r1) return;
    uint32_t v[K2P2W_ITEMS], m[K2P2W_ITEMS], nn[K2P2W_ITEMS], rs[K2P2W_ITEMS];
#pragma unroll
    for (int j = 0; j < K2P2W_ITEMS; j++) {
        const bool ok = i0 + j < r1;
        v[j] = ok ? p.rec_v[i0 + j] : 1u; m[j] = ok ? p.rec_m[i0 + j] : 0u; nn[j] = ok ? p.rec_n[i0 + j] : 0u;
    }
#pragma unroll
    for (int j = 0; j < K2P2W_ITEMS; j++) rs[j] = p.rssi[m[j]];
    /* the register in front of record i0: the bits since the last reset, zero-extended */
    uint32_t sr = 0, pend = 0;
    if (!(v[0] & 1u)) {
        uint32_t have = 0;
        uint64_t k = i0;
        while (true) {
            if (k == 0) {                                            /* start of the batch: the carried state */
                const RlState c = *p.carry;
                sr |= c.sr << have;
                if (i0 == 0) pend = (c.flags >> 1) & 1u;
                break;
            }
            k--;
            const uint32_t pv = p.rec_v[k], pn = p.rec_n[k];
            const uint32_t take = pn < 16u - have ? pn : 16u - have;
            if (pv & 2u) sr |= ((1u << take) - 1u) << have;
            have += take;
            if (have >= 16u || (pv & 1u)) break;                     /* nothing older than a reset counts */
        }
        sr &= 0xFFFFu;
    }
    uint64_t ord = p.base[lane] + part[tid];
#pragma unroll
    for (int j = 0; j < K2P2W_ITEMS; j++) {
        if (i0 + j >= r1) break;
        if (v[j] & 1u) { sr = 0; pend = 1; }
        const uint32_t level = (v[j] >> 1) & 1u;
        const uint64_t head = ((uint64_t)(p.m_base + m[j]) << 24) | ((uint64_t)rs[j] << 16) | level;
        for (uint32_t k = 0; k < nn[j]; k++) {
            sr = ((sr << 1) | level) & 0xFFFFu;
            const uint32_t sync = ac_match<ChainT1C1>(sr, p.ac_err);
            p.ring[ord & p.ring_mask] = head | (pend << 2) | (sync << 1);
            pend = 0;
            if (sync) {
#ifdef WMB_HOSTSIM
                const uint32_t slot = p.sd->n_cand++;
#else
                const uint32_t slot = atomicAdd(&p.sd->n_cand, 1u);
#endif
                if (slot < p.cand_cap) p.cand[slot] = ord;
                else p.sd->cand_overflow = 1;
            }
            ord++;
        }
        if (i0 + j + 1 == N) {                                       /* the last record of the batch */
            p.p2_out->sr = sr; p.p2_out->flags = pend << 1; p.p2_out->run = 1;
        }
    }
}

/* end of batch: compose the carried RlState from phase 1's end state (raw bits, level, run,
 * "reset since the last record") and phase 2's state after the last record */
WMB_D void k2p_fold(const P1State *p1_end, RlState *p2_out, RlState *carry, const K2pDev *pd, const RlState *mono_end,
                    uint32_t *stat_fallbacks)
{
    if (pd->fallback) {                 /* the batch was redone with the monolithic lanes: their end state carries */
        *carry = *mono_end;
        p2_out->run = 0;
        (*stat_fallbacks)++;
        return;
    }
    RlState c = *carry;
    if (p2_out->run) { c.a = p2_out->a; c.b = p2_out->b; c.sr = p2_out->sr; }
    c.raw = p1_end->raw; c.run = p1_end->run;
    if (p1_end->pend) { c.a = 8 * 256; c.b = 0; c.sr = 0; }      /* runlength_algorithm_reset_t1_c1 */
    c.flags = (p1_end->level & 1u) | ((p1_end->pend & 1u) << 1);
    *carry = c;
    p2_out->run = 0;
}
