/*
 * wmb_spectrum.cuh -- the band survey (wmb_set_spectrum / wmb_take_spectrum, DESIGN.md §8): a power spectrum of the raw
 * cu8 input over the whole captured band, mean and peak hold per record, to find the carriers worth decoding.
 *
 * The definition (normative; tests/spectrum_cases.py restates it in numpy) is in include/wmbus_b200.h.  In short: block
 * b is global IQ samples [b N, (b + 1) N); per block, every step a separately rounded fp32 operation:
 *   i = (int)(u - 127.5f) per byte, x = ((float)i_I * hann[n], (float)i_Q * hann[n]),
 *   X = radix-2 decimation-in-time FFT on bit-reversed input, twiddle tw[j N / 2^s] at stage s, butterfly j:
 *       t = (w_re b_re - w_im b_im, w_re b_im + w_im b_re), a' = a + t, b' = a - t,
 *   p = re re + im im;
 * record r (blocks [r B, (r + 1) B)) holds per fftshifted bin sum = sum of rint(p) (uint64, exact in any order) and
 * peak = max p (exact in any order; as bit patterns, an integer max).
 *
 * Per batch, on the demod stream right behind the demod kernel, while it still owns the input bytes:
 *   ks_fft_kernel    a CTA per unit: a run of at most G blocks of one record.  2048 / N blocks side by side per pass
 *                    (2048 points, 256 threads x 8 samples, one 128-bit load each), converted, windowed and stored
 *                    bit-reversed in shared memory; two radix-2 stages per pass in registers, a last single stage when
 *                    log2 N is odd; each thread keeps the sums and maxima of its 8 points in registers over the unit,
 *                    then one atomicAdd / atomicMax per bin and CTA into the record's row of the ring
 *   ks_close_kernel  the rows the batch closes -> the batch's result slot, and zeroed in the ring
 * The ring holds a row per record that can be open at once: a batch touches the record left open by the last block
 * pushed before it and the records of its own blocks, at most batch_blocks / B + 2 consecutive ones.
 */
#pragma once

#define WMB_SPEC_THREADS 256u              /* threads of ks_fft_kernel                                           */
#define WMB_SPEC_POINTS  2048u             /* points per pass: WMB_SPEC_POINTS / N blocks side by side            */
#define WMB_SPEC_PER_T   (WMB_SPEC_POINTS / WMB_SPEC_THREADS)   /* 8: samples per thread, one 16-byte load          */
#define WMB_SPEC_MAXN    2048u

struct SpecParams {
    const uint8_t *in;              /* the batch's bytes: byte 0 is IQ sample b_first * N                         */
    int64_t  b_first;               /* global index of the batch's first block                                    */
    int64_t  c0, c1;                /* blocks counted by this batch, [c0, c1) (global)                            */
    int64_t  g_lo;                  /* first unit (global: record * U + block-in-record / G)                      */
    uint32_t n_units;
    uint32_t N, logN, B, G, U;      /* U = ceil(B / G) units per record                                           */
    uint32_t R;                     /* ring rows                                                                  */
    const float *hann;              /* [N]                                                                        */
    const float *tw;                /* [N / 2][2]: (cos, -sin)                                                    */
    uint64_t *sum;                  /* ring [R][N], fftshifted bins                                               */
    uint32_t *peak;                 /* ring [R][N], float bit patterns                                            */
};

struct SpecSmem {
    union {
        struct { float re[WMB_SPEC_POINTS], im[WMB_SPEC_POINTS]; };
        uint64_t red[WMB_SPEC_POINTS];  /* end of a unit: per-point sums, then per-point maxima                   */
    };
    float tw_re[WMB_SPEC_MAXN / 2], tw_im[WMB_SPEC_MAXN / 2];
    float hann[WMB_SPEC_MAXN];
};

struct SpecAcc {                    /* one thread's registers: its 8 points (t + 256 k) over a unit */
    uint64_t sum[WMB_SPEC_PER_T];
    float peak[WMB_SPEC_PER_T];
};

struct SpecUnit { int64_t rec, ba, bb; };           /* unit -> record, blocks [ba, bb) */

WMB_HD SpecUnit spec_unit(const SpecParams &p, int64_t g)
{
    SpecUnit u;
    u.rec = g / p.U;
    const int64_t j = g % p.U;
    int64_t a = u.rec * p.B + j * p.G, b = a + p.G;
    if (b > (u.rec + 1) * (int64_t)p.B) b = (u.rec + 1) * (int64_t)p.B;
    u.ba = a > p.c0 ? a : p.c0;
    u.bb = b < p.c1 ? b : p.c1;
    return u;
}

WMB_D void ks_tables(const SpecParams &p, SpecSmem &sm, uint32_t t)
{
    for (uint32_t k = t; k < p.N; k += WMB_SPEC_THREADS) sm.hann[k] = p.hann[k];
    for (uint32_t k = t; k < p.N / 2; k += WMB_SPEC_THREADS) { sm.tw_re[k] = p.tw[2 * k]; sm.tw_im[k] = p.tw[2 * k + 1]; }
}

WMB_D void ks_acc_clear(SpecAcc &a)
{
#pragma unroll
    for (uint32_t k = 0; k < WMB_SPEC_PER_T; k++) { a.sum[k] = 0; a.peak[k] = 0.f; }
}

/* The phase functions take L = log2 N as an argument: the kernel is instantiated per N, so every division, modulo and
 * stage count below is a shift or a mask of a constant; the CPU build passes p.logN. */

/* thread t: samples [8 t, 8 t + 8) of the pass -> block ba + pass * (2048 / N) + 8 t / N, converted, windowed, stored at
 * their bit-reversed places inside the block */
WMB_D void ks_load(const SpecParams &p, SpecSmem &sm, const SpecUnit &u, int64_t pass, uint32_t t, uint32_t L)
{
    const uint32_t pt = WMB_SPEC_PER_T * t, s = pt >> L, n0 = pt & ((1u << L) - 1u);
    const int64_t b = u.ba + (pass << (11 - L)) + s;
    uint32_t w[4] = {0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u};      /* (a block past the unit: zeros) */
    if (b < u.bb) {
        const uint8_t *src = p.in + (((size_t)(b - p.b_first)) << (L + 1)) + 2 * n0;
#ifdef WMB_HOSTSIM
        memcpy(w, src, 16);
#else
        const uint4 q = *(const uint4 *)src;
        w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
#endif
    }
#pragma unroll
    for (uint32_t k = 0; k < WMB_SPEC_PER_T; k++) {
        const uint32_t n = n0 + k;
        const float h = sm.hann[n];
        const uint32_t uI = (w[k >> 1] >> (16 * (k & 1))) & 0xFFu, uQ = (w[k >> 1] >> (16 * (k & 1) + 8)) & 0xFFu;
        const int iI = (int)wmb_fsub((float)uI, 127.5f), iQ = (int)wmb_fsub((float)uQ, 127.5f);
        const uint32_t at = (s << L) + (wmb_brev(n) >> (32 - L));
        sm.re[at] = wmb_fmul((float)iI, h);
        sm.im[at] = wmb_fmul((float)iQ, h);
    }
}

/* a = a + w b, b = a - w b, every operation rounded on its own */
WMB_D void ks_bfly(float &ar, float &ai, float &br, float &bi, float wr, float wi)
{
    const float tr = wmb_fsub(wmb_fmul(wr, br), wmb_fmul(wi, bi));
    const float ti = wmb_fadd(wmb_fmul(wr, bi), wmb_fmul(wi, br));
    const float xr = ar, xi = ai;
    ar = wmb_fadd(xr, tr); ai = wmb_fadd(xi, ti);
    br = wmb_fsub(xr, tr); bi = wmb_fsub(xi, ti);
}

/* stages s and s + 1 (half h = 2^lh = 2^(s-1)): thread t takes the groups q = t, t + 256 of 4 points
 * (base + j + {0, h, 2h, 3h}); twiddles tw[j N / 2h] and tw[j N / 4h], tw[(j + h) N / 4h] */
WMB_D void ks_stage2(SpecSmem &sm, uint32_t lh, uint32_t L, uint32_t t)
{
    const uint32_t h = 1u << lh, s1 = L - lh - 1, s2 = L - lh - 2;
#pragma unroll
    for (uint32_t q = t; q < WMB_SPEC_POINTS / 4; q += WMB_SPEC_THREADS) {
        const uint32_t j = q & (h - 1u), base = ((q >> lh) << (lh + 2)) + j;
        float r0 = sm.re[base], i0 = sm.im[base], r1 = sm.re[base + h], i1 = sm.im[base + h];
        float r2 = sm.re[base + 2 * h], i2 = sm.im[base + 2 * h], r3 = sm.re[base + 3 * h], i3 = sm.im[base + 3 * h];
        const float w1r = sm.tw_re[j << s1], w1i = sm.tw_im[j << s1];
        ks_bfly(r0, i0, r1, i1, w1r, w1i);
        ks_bfly(r2, i2, r3, i3, w1r, w1i);
        ks_bfly(r0, i0, r2, i2, sm.tw_re[j << s2], sm.tw_im[j << s2]);
        ks_bfly(r1, i1, r3, i3, sm.tw_re[(j + h) << s2], sm.tw_im[(j + h) << s2]);
        sm.re[base] = r0; sm.im[base] = i0; sm.re[base + h] = r1; sm.im[base + h] = i1;
        sm.re[base + 2 * h] = r2; sm.im[base + 2 * h] = i2; sm.re[base + 3 * h] = r3; sm.im[base + 3 * h] = i3;
    }
}

/* the last stage alone (log2 N odd): half h = 2^lh = N / 2 */
WMB_D void ks_stage1(SpecSmem &sm, uint32_t lh, uint32_t L, uint32_t t)
{
    const uint32_t h = 1u << lh, s1 = L - lh - 1;
#pragma unroll
    for (uint32_t q = t; q < WMB_SPEC_POINTS / 2; q += WMB_SPEC_THREADS) {
        const uint32_t j = q & (h - 1u), base = ((q >> lh) << (lh + 1)) + j;
        float r0 = sm.re[base], i0 = sm.im[base], r1 = sm.re[base + h], i1 = sm.im[base + h];
        ks_bfly(r0, i0, r1, i1, sm.tw_re[j << s1], sm.tw_im[j << s1]);
        sm.re[base] = r0; sm.im[base] = i0; sm.re[base + h] = r1; sm.im[base + h] = i1;
    }
}

/* the blocks of this pass that lie in the unit (the rest of the 2048 / N side by side are not counted) */
WMB_D uint32_t ks_pass_blocks(const SpecUnit &u, int64_t pass, uint32_t L)
{
    const int64_t left = u.bb - (u.ba + (pass << (11 - L)));
    return left < ((int64_t)1 << (11 - L)) ? (uint32_t)left : (1u << (11 - L));
}

/* thread t: the power of its points t + 256 k, into its registers */
WMB_D void ks_power(const SpecSmem &sm, uint32_t nvalid, uint32_t t, SpecAcc &a, uint32_t L)
{
#pragma unroll
    for (uint32_t k = 0; k < WMB_SPEC_PER_T; k++) {
        const uint32_t pt = t + WMB_SPEC_THREADS * k;
        if ((pt >> L) >= nvalid) continue;
        const float re = sm.re[pt], im = sm.im[pt];
        const float pw = wmb_fadd(wmb_fmul(re, re), wmb_fmul(im, im));
#ifdef WMB_HOSTSIM
        a.sum[k] += (uint64_t)llrintf(pw);
#else
        a.sum[k] += __float2ull_rn(pw);
#endif
        a.peak[k] = pw > a.peak[k] ? pw : a.peak[k];
    }
}

/* end of a unit: the registers -> shared memory (sums, or maxima as bit patterns), then per bin over the blocks side by
 * side -> one atomic per bin into the record's ring row */
WMB_D void ks_red_put(SpecSmem &sm, const SpecAcc &a, uint32_t t, bool peaks)
{
#pragma unroll
    for (uint32_t k = 0; k < WMB_SPEC_PER_T; k++)
        sm.red[t + WMB_SPEC_THREADS * k] = peaks ? (uint64_t)wmb_f2u(a.peak[k]) : a.sum[k];
}

WMB_D void ks_red_flush(const SpecParams &p, const SpecSmem &sm, const SpecUnit &u, uint32_t t, bool peaks, uint32_t L)
{
    const uint32_t N = 1u << L;
    const size_t row = (size_t)(u.rec % p.R) << L;
    for (uint32_t k = t; k < N; k += WMB_SPEC_THREADS) {
        uint64_t v = 0;
        for (uint32_t s = 0; s < (WMB_SPEC_POINTS >> L); s++) {
            const uint64_t x = sm.red[(s << L) + k];
            v = peaks ? (x > v ? x : v) : v + x;
        }
        const uint32_t bin = (k + N / 2) & (N - 1u);      /* fftshift: bin 0 is -fs / 2 */
        if (!v) continue;
#ifdef WMB_HOSTSIM
        if (peaks) { if ((uint32_t)v > p.peak[row + bin]) p.peak[row + bin] = (uint32_t)v; }
        else p.sum[row + bin] += v;
#else
        if (peaks) atomicMax(p.peak + row + bin, (uint32_t)v);
        else atomicAdd((unsigned long long *)(p.sum + row + bin), (unsigned long long)v);
#endif
    }
}

/* the rows a batch closes: slot row j <- ring row of record (j == 0 && lone >= 0 ? lone : r_lo + j - (lone >= 0)), which
 * is zeroed for the record that will use it next */
struct SpecCloseParams {
    uint64_t *sum; uint32_t *peak;  /* ring */
    uint64_t *out_sum; uint32_t *out_peak;    /* the slot's rows */
    int64_t lone, r_lo;
    uint32_t n, N, R;
};

WMB_D void ks_close(const SpecCloseParams &p, uint32_t j, uint32_t k)
{
    const int64_t rec = (j == 0 && p.lone >= 0) ? p.lone : p.r_lo + (int64_t)j - (p.lone >= 0 ? 1 : 0);
    const size_t at = (size_t)(rec % p.R) * p.N + k, to = (size_t)j * p.N + k;
    p.out_sum[to] = p.sum[at]; p.out_peak[to] = p.peak[at];
    p.sum[at] = 0; p.peak[at] = 0;
}

#ifndef WMB_HOSTSIM
template <uint32_t L>
__global__ void __launch_bounds__(WMB_SPEC_THREADS) ks_fft_kernel(const SpecParams p)
{
    __shared__ SpecSmem sm;
    const uint32_t t = threadIdx.x;
    ks_tables(p, sm, t);
    SpecAcc a;
    for (int64_t gi = blockIdx.x; gi < (int64_t)p.n_units; gi += gridDim.x) {
        const SpecUnit u = spec_unit(p, p.g_lo + gi);
        ks_acc_clear(a);
        const int64_t passes = (u.bb - u.ba + (1 << (11 - L)) - 1) >> (11 - L);
        for (int64_t pass = 0; pass < passes; pass++) {
            __syncthreads();                               /* the tables / the last pass's reads are done */
            ks_load(p, sm, u, pass, t, L);
            __syncthreads();
#pragma unroll
            for (uint32_t lh = 0; lh + 2 <= L; lh += 2) { ks_stage2(sm, lh, L, t); __syncthreads(); }
            if (L & 1u) { ks_stage1(sm, L - 1, L, t); __syncthreads(); }
            ks_power(sm, ks_pass_blocks(u, pass, L), t, a, L);
        }
        __syncthreads();
        ks_red_put(sm, a, t, false);
        __syncthreads();
        ks_red_flush(p, sm, u, t, false, L);
        __syncthreads();
        ks_red_put(sm, a, t, true);
        __syncthreads();
        ks_red_flush(p, sm, u, t, true, L);
    }
}

__global__ void ks_close_kernel(const SpecCloseParams p)
{
    for (uint32_t k = threadIdx.x; k < p.N; k += blockDim.x) ks_close(p, blockIdx.x, k);
}
#endif
