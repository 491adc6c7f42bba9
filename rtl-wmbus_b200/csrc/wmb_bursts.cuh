/*
 * wmb_bursts.cuh -- the burst report (wmb_set_bursts / wmb_take_bursts, DESIGN.md §8): every stretch of a chain's
 * (unsigned)rssi at or above a level, decoded or not, with its level and carrier offset.
 *
 * Per enabled chain and batch, on cs behind the demod kernel (the set's rssi / dphi, history prefix included):
 *   kb_mask     thread per 32-sample word: rssi >= level -> mask word (samples before the first one pushed are below)
 *   kb_events   thread per 128-sample unit: run starts (an above sample with none in the G before it) and run ends
 *               (an above sample followed by G below ones), counted, then -- after a count scan -- written in order
 *   kb_runs     one block: the k-th start paired with the k-th end (the run open at the last batch end first), the cut
 *               grid applied (multiples of P at least Q after the run start), pieces >= Lmin listed in start order
 *   kb_reduce   block per piece: rssi sum / peak and the carrier-offset window sum, integer arithmetic (exact in any
 *               order); the piece still open at the batch end leaves its partial sums in BurstDev
 * A run end is decided G samples after its last above sample, so an end that lands in the next batch reads back into
 * the set's history prefix (G <= 196 samples, the prefix holds >= 1536).  No piece is longer than Q + P, so no sum
 * reaches further back than the open piece's partial sums, which cover [piece start, last above sample + 1).
 */
#pragma once

#define WMB_BURST_Q      (1ll << 17)       /* a run is cut only at least Q samples after its start            */
#define WMB_BURST_P      (1ll << 16)       /* ... at multiples of P (global decimated index)                   */
#define WMB_BURST_UNIT   128u              /* samples per thread of kb_events                                  */
#define WMB_BURST_LOOK   8u                /* mask words kept before batch sample 0: >= G + 32 samples         */
#define WMB_BURST_BLOCK  256u              /* threads of kb_runs / kb_reduce                                   */

#define WMB_BURST_F_CONTINUED 1u           /* the piece starts at a cut                                        */
#define WMB_BURST_F_CUT       2u           /* the piece ends at a cut                                          */
#define WMB_BURST_F_AT_END    4u           /* the input ended before the run did                               */

/* per chain: bridge G, least reported length Lmin, offset window [start + g0, start + g0 + w) (8 / 32 nominal chips) */
WMB_HD int64_t burst_G(uint32_t ch) { return ch == 0 ? 64 : 196; }
WMB_HD int64_t burst_Lmin(uint32_t ch) { return ch == 0 ? 256 : 782; }
WMB_HD int64_t burst_g0(uint32_t ch) { return ch == 0 ? 64 : 196; }
WMB_HD int64_t burst_w(uint32_t ch) { return ch == 0 ? 256 : 781; }

struct BurstDev {                   /* carried from batch to batch, one per chain (absolute sample indices) */
    int64_t  s, ps, la;             /* open run: its start, the open piece's start, the last above sample         */
    uint64_t rsum;                  /* open piece: rssi sum, window sum, peak, window samples over [ps, la + 1)  */
    int64_t  wsum;
    uint32_t peak, wn;
    uint32_t open, flags;           /* a run is in progress; the open piece's flags                               */
    uint64_t n_ev;                  /* events of the current batch (the count scan's total)                       */
    uint32_t n_items, pad;
    QualAcc  q;                     /* quality: the open piece's class sums, once its window is whole (qdone)     */
    uint32_t qdone, pad2;
};

struct BurstItem {                  /* one piece for kb_reduce, batch-relative sample indices */
    int64_t  a, b;                  /* the samples summed here                                                    */
    int64_t  ps, pe;                /* the piece (pe: its end; the open piece: b)                                 */
    uint64_t rsum; int64_t wsum;    /* sums before a (the open piece of the last batch)                           */
    uint32_t peak, wn;
    uint32_t flags; int32_t out;    /* out: record index, -1: the piece still open (sums go to BurstDev)          */
    QualAcc  q;                     /* quality sums taken in an earlier batch (qdone)                             */
    uint32_t qdone, pad;
};

/* what kb_reduce's quality pass does for one item: the window [lo, hi) with its sum and n, run = take the sums now */
struct BurstQPlan { int64_t lo, hi, sum, n; uint32_t run, pad; };

struct BurstRec {                   /* device -> host, one per reported piece */
    uint64_t start, end;
    uint64_t rssi_sum;
    int64_t  sum;
    uint32_t n;
    uint8_t  peak, chain, flags, pad;
};

struct BurstSlot {                  /* per result slot: records per chain, and where a chain's next piece may start */
    uint32_t n[WMB_N_CHAINS];
    uint32_t open[WMB_N_CHAINS];
    int64_t  ps[WMB_N_CHAINS];
};

struct BurstParams {
    const uint8_t *rssi;            /* batch sample 0 of the set (the history prefix lies before it)              */
    const float *dphi;
    int64_t  M;                     /* batch samples; 0: the end-of-input gather                                  */
    int64_t  clip;                  /* samples before sample 0 that exist since the last reset / seek            */
    int64_t  m_first;               /* absolute index of batch sample 0                                           */
    uint32_t level, chain, final_;
    uint32_t nw, units;             /* mask words of the batch, kb_events units                                   */
    uint32_t *mask;                 /* [WMB_BURST_LOOK + nw]                                                      */
    uint32_t *cnt; uint64_t *base;  /* [units]                                                                    */
    int64_t  *ev;                   /* events: 2 * start, or 2 * end + 1 (batch-relative)                        */
    BurstDev *bd;
    BurstItem *items;
    BurstRec *out;                  /* this slot's records of the chain                                           */
    BurstSlot *slot;
    QualAcc  *qout;                 /* quality (null: off): the records' class sums, parallel to out              */
    uint32_t qual_skip, pad;        /* 1 (-a): zero sums                                                          */
};

WMB_D int burst_msb(uint32_t v)
{
#ifdef WMB_HOSTSIM
    return 31 - __builtin_clz(v);
#else
    return 31 - __clz((int)v);
#endif
}

WMB_D void kb_load32(const uint8_t *p, uint32_t w[8])
{
#ifdef WMB_HOSTSIM
    memcpy(w, p, 32);
#else
    const uint4 a = ((const uint4 *)p)[0], b = ((const uint4 *)p)[1];
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
#endif
}

/* mask word wi = batch samples [32 (wi - LOOK), +32) */
WMB_D void kb_mask(const BurstParams &p, uint32_t wi)
{
    const int64_t m0 = 32 * ((int64_t)wi - (int64_t)WMB_BURST_LOOK);
    uint32_t w[8];
    kb_load32(p.rssi + m0, w);
    uint32_t bits = 0;
#pragma unroll
    for (int k = 0; k < 32; k++) bits |= (((w[k >> 2] >> (8 * (k & 3))) & 0xFFu) >= p.level ? 1u : 0u) << k;
    const int64_t lo = -p.clip - m0, hi = p.M - m0;             /* valid bits [lo, hi) */
    if (lo > 0) bits = lo >= 32 ? 0u : bits & ~((1u << lo) - 1u);
    if (hi < 32) bits = hi <= 0 ? 0u : bits & ((1u << hi) - 1u);
    p.mask[wi] = bits;
}

/* the events decided in unit u (samples [128 u, 128 u + 128)): a start at m, or the end e = la + 1 decided at
 * m = la + G.  write: store them at ev[base[u]...]; returns their number */
WMB_D uint32_t kb_events(const BurstParams &p, uint32_t u, bool write)
{
    const int64_t G = burst_G(p.chain);
    const int64_t m0 = (int64_t)u * WMB_BURST_UNIT;
    const int64_t far = -((int64_t)1 << 40);
    int64_t la = far;                                         /* last above sample before m0 (only <= G back matters) */
    for (int64_t k = 1; k <= (int64_t)WMB_BURST_LOOK; k++) {
        const uint32_t mw = p.mask[WMB_BURST_LOOK + (m0 >> 5) - k];
        if (mw) { la = m0 - 32 * k + burst_msb(mw); break; }
    }
    const int64_t end = m0 + WMB_BURST_UNIT < p.M ? m0 + WMB_BURST_UNIT : p.M;
    int64_t *out = write ? p.ev + p.base[u] : nullptr;
    uint32_t n = 0;
    for (int64_t w0 = m0; w0 < end; w0 += 32) {
        const uint32_t mw = p.mask[WMB_BURST_LOOK + (w0 >> 5)];
        if (!mw && w0 - la > G) continue;                     /* nothing starts or ends in a quiet word */
        const int64_t we = w0 + 32 < end ? w0 + 32 : end;
        for (int64_t m = w0; m < we; m++) {
            if ((mw >> (m - w0)) & 1u) {
                if (m - la > G) { if (write) out[n] = 2 * m; n++; }
                la = m;
            } else if (m - la == G) {
                if (write) out[n] = 2 * (la + 1) + 1;
                n++;
            }
        }
    }
    return n;
}

/* kb_runs: run item i of the batch (the run open at the last batch end is item 0), its pieces.
 * For each piece >= Lmin and the piece still open at the batch end: one BurstItem (emit) */
struct BurstRunCtx {                /* what every thread of kb_runs reads before anything is written */
    int64_t s0, ps0, la0, la;       /* batch-relative: carried run start / piece start / last above; this batch's la */
    uint64_t rsum; int64_t wsum; uint32_t peak, wn, flags0;
    uint32_t open_in, n_runs;
    uint64_t n_ev;
    QualAcc q; uint32_t qdone;
};

WMB_D void kb_run_ctx(const BurstParams &p, BurstRunCtx &r)
{
    const BurstDev &bd = *p.bd;
    r.open_in = bd.open;
    r.n_ev = p.final_ ? 0 : bd.n_ev;
    r.s0 = bd.s - p.m_first; r.ps0 = bd.ps - p.m_first; r.la0 = bd.la - p.m_first;
    r.rsum = bd.rsum; r.wsum = bd.wsum; r.peak = bd.peak; r.wn = bd.wn; r.flags0 = bd.flags;
    r.q = bd.q; r.qdone = bd.qdone;
    /* the last above sample so far: an open run has one within the last G samples */
    r.la = r.open_in ? r.la0 : -((int64_t)1 << 40);
    const int64_t G = burst_G(p.chain);
    if (p.M > 0) {
        int64_t wlo = ((p.M - G) >> 5) - 1;
        if (wlo < -(int64_t)WMB_BURST_LOOK) wlo = -(int64_t)WMB_BURST_LOOK;
        for (int64_t w = ((p.M - 1) >> 5); w >= wlo; w--) {
            const uint32_t mw = p.mask[WMB_BURST_LOOK + w];
            if (mw) { const int64_t m = 32 * w + burst_msb(mw); if (m > r.la) r.la = m; break; }
        }
    }
    const uint64_t rest = r.open_in ? (r.n_ev ? r.n_ev - 1 : 0) : r.n_ev;
    r.n_runs = (uint32_t)(r.open_in + (rest + 1) / 2);
}

WMB_HD int64_t burst_grid_up(int64_t abs_m)          /* least multiple of P >= abs_m (abs_m >= 0) */
{
    return (abs_m + WMB_BURST_P - 1) / WMB_BURST_P * WMB_BURST_P;
}

/* run item i -> its pieces.  write == false: returns the number of BurstItems; write: stores them from items[at] */
WMB_D uint32_t kb_run(const BurstParams &p, const BurstRunCtx &r, uint32_t i, bool write, uint32_t at)
{
    const int64_t Lmin = burst_Lmin(p.chain);
    int64_t s, ps, a0;                                        /* run start, first piece start, first sample summed here */
    uint32_t fl;
    bool closed, at_end = false;
    int64_t e;                                                /* closed: the run end; open: last above + 1 */
    uint64_t rsum = 0; int64_t wsum = 0; uint32_t peak = 0, wn = 0;
    const uint64_t j0 = r.open_in ? 1 : 0;
    if (r.open_in && i == 0) {
        s = r.s0; ps = r.ps0; fl = r.flags0; a0 = r.la0 + 1;
        rsum = r.rsum; wsum = r.wsum; peak = r.peak; wn = r.wn;
        if (r.n_ev) { closed = true; e = p.ev[0] >> 1; }
        else if (p.final_) { closed = true; at_end = true; e = r.la0 + 1; }
        else { closed = false; e = r.la + 1; }
    } else {
        const uint64_t k = j0 + 2 * (uint64_t)(i - r.open_in);
        s = p.ev[k] >> 1; ps = s; fl = 0; a0 = s;
        if (k + 1 < r.n_ev) { closed = true; e = p.ev[k + 1] >> 1; }
        else { closed = false; e = r.la + 1; }
    }
    /* cuts: multiples of P at least Q after the run start; the open run's only as far as its last above sample */
    const int64_t first = (s + WMB_BURST_Q > ps + 1 ? s + WMB_BURST_Q : ps + 1) + p.m_first;
    int64_t c = burst_grid_up(first) - p.m_first;
    uint32_t n = 0;
    int64_t cur = ps;
    for (;; c += WMB_BURST_P) {
        const bool is_cut = c < e;                            /* closed: c < e; open: c <= la, i.e. c < la + 1 = e */
        const int64_t pe = is_cut ? c : e;
        const bool last = !is_cut;
        const bool item_open = last && !closed;
        const uint32_t f = fl | (is_cut ? WMB_BURST_F_CUT : 0u) | (last && at_end ? WMB_BURST_F_AT_END : 0u);
        if (item_open || pe - cur >= Lmin) {
            if (write) {
                BurstItem it;
                it.a = cur > a0 ? cur : a0; it.b = pe; it.ps = cur; it.pe = pe;
                const bool carried = cur == ps && r.open_in && i == 0;
                it.rsum = carried ? rsum : 0; it.wsum = carried ? wsum : 0;
                it.peak = carried ? peak : 0; it.wn = carried ? wn : 0;
                if (carried) it.q = r.q; else qual_zero(it.q);
                it.qdone = carried ? r.qdone : 0u; it.pad = 0;
                it.flags = f; it.out = item_open ? -1 : (int32_t)(at + n);
                p.items[at + n] = it;
            }
            n++;
        }
        if (last) break;
        cur = c; fl = WMB_BURST_F_CONTINUED;
    }
    return n;
}

/* kb_runs over chunks of WMB_BURST_BLOCK run items: count (thread t), scan (one thread), write (thread t) */
WMB_D void kb_runs_count(const BurstParams &p, const BurstRunCtx &r, uint32_t chunk, uint32_t t, uint32_t *cnt)
{
    const uint32_t i = chunk * WMB_BURST_BLOCK + t;
    cnt[t] = i < r.n_runs ? kb_run(p, r, i, false, 0) : 0u;
}
WMB_D void kb_runs_scan(uint32_t *cnt, uint32_t *total)
{
    uint32_t acc = *total;
    for (uint32_t t = 0; t < WMB_BURST_BLOCK; t++) { const uint32_t v = cnt[t]; cnt[t] = acc; acc += v; }
    *total = acc;
}
WMB_D void kb_runs_write(const BurstParams &p, const BurstRunCtx &r, uint32_t chunk, uint32_t t, const uint32_t *at)
{
    const uint32_t i = chunk * WMB_BURST_BLOCK + t;
    if (i < r.n_runs) kb_run(p, r, i, true, at[t]);
}
/* the new carried run and the slot's summary (one thread, after the last chunk) */
WMB_D void kb_runs_finish(const BurstParams &p, const BurstRunCtx &r, uint32_t n_items)
{
    BurstDev &bd = *p.bd;
    bd.n_items = n_items;
    const BurstItem *last = n_items ? &p.items[n_items - 1] : nullptr;
    const bool open = last && last->out < 0;
    uint32_t n_out = open ? n_items - 1 : n_items;
    if (open) {
        /* the open piece belongs to the last run: its start is the last start event, or the carried run's */
        int64_t s = r.s0;
        const uint64_t j0 = r.open_in ? 1 : 0;
        if (!(r.open_in && r.n_runs == 1)) s = p.ev[j0 + 2 * (uint64_t)(r.n_runs - 1 - r.open_in)] >> 1;
        bd.s = s + p.m_first; bd.ps = last->ps + p.m_first; bd.la = r.la + p.m_first; bd.flags = last->flags;
    }
    bd.open = open ? 1u : 0u;
    p.slot->n[p.chain] = n_out;
    p.slot->open[p.chain] = bd.open;
    p.slot->ps[p.chain] = open ? bd.ps : 0;
}

struct BurstPart { uint64_t rsum; int64_t wsum; uint32_t peak, pad; };

/* kb_reduce: thread t of nt over item it */
WMB_D void kb_reduce_part(const BurstParams &p, uint32_t it, uint32_t t, uint32_t nt, BurstPart *part)
{
    const BurstItem &x = p.items[it];
    uint64_t rsum = 0;
    uint32_t peak = 0;
    for (int64_t m = x.a + t; m < x.b; m += nt) {
        const uint32_t v = p.rssi[m];
        rsum += v;
        peak = v > peak ? v : peak;
    }
    const int64_t wlo0 = x.ps + burst_g0(p.chain), whi0 = x.ps + burst_g0(p.chain) + burst_w(p.chain);
    const int64_t wlo = wlo0 > x.a ? wlo0 : x.a;
    const int64_t whi = whi0 < x.b ? whi0 : x.b;
    int64_t wsum = 0;
    for (int64_t m = wlo + t; m < whi; m += nt) wsum += wmb_ofs_x(p.dphi[m]);
    part[t].rsum = rsum; part[t].wsum = wsum; part[t].peak = peak; part[t].pad = 0;
}

/* qp (quality on): the item's quality pass.  The window [ps + g0, min(pe, ps + g0 + w)) is whole once its end is known:
 * a closed piece's always, the open piece's when ps + g0 + w <= b (its end lies at or after b).  The sums are taken in
 * that batch; the window reaches back at most G + w + 1 samples before it, inside the set's history prefix */
WMB_D void kb_reduce_finish(const BurstParams &p, uint32_t it, const BurstPart *part, uint32_t nt, BurstQPlan *qp)
{
    const BurstItem &x = p.items[it];
    uint64_t rsum = x.rsum;
    int64_t wsum = x.wsum;
    uint32_t peak = x.peak;
    for (uint32_t t = 0; t < nt; t++) { rsum += part[t].rsum; wsum += part[t].wsum; peak = part[t].peak > peak ? part[t].peak : peak; }
    const int64_t wlo0 = x.ps + burst_g0(p.chain), whi0 = x.ps + burst_g0(p.chain) + burst_w(p.chain);
    const int64_t wlo = wlo0 > x.a ? wlo0 : x.a;
    const int64_t whi = whi0 < x.b ? whi0 : x.b;
    const uint32_t wn = x.wn + (uint32_t)(whi > wlo ? whi - wlo : 0);
    if (qp) {
        const int64_t qhi = x.out < 0 ? whi0 : (whi0 < x.pe ? whi0 : x.pe);
        qp->lo = wlo0; qp->hi = qhi; qp->sum = wsum; qp->n = wn; qp->pad = 0;
        qp->run = (!x.qdone && !p.qual_skip && (x.out >= 0 || whi0 <= x.b)) ? 1u : 0u;
    }
    if (x.out < 0) {
        BurstDev &bd = *p.bd;
        bd.rsum = rsum; bd.wsum = wsum; bd.peak = peak; bd.wn = wn;
        return;
    }
    BurstRec r;
    r.start = (uint64_t)(x.ps + p.m_first); r.end = (uint64_t)(x.pe + p.m_first);
    r.rssi_sum = rsum; r.sum = wsum; r.n = wn;
    r.peak = (uint8_t)peak; r.chain = (uint8_t)p.chain; r.flags = (uint8_t)x.flags; r.pad = 0;
    p.out[x.out] = r;
}

/* the quality pass (quality on, after kb_reduce_finish): thread t of nt */
WMB_D void kb_qual_part(const BurstParams &p, const BurstQPlan &qp, uint32_t t, uint32_t nt, QualAcc *part)
{
    if (qp.run) qual_part(p.dphi, qp.lo, qp.hi, qp.sum, qp.n, t, nt, part[t]);
    else qual_zero(part[t]);
}

/* ... and its result: the record's sums, or the open piece's (kept in BurstDev until its record is written) */
WMB_D void kb_qual_finish(const BurstParams &p, uint32_t it, const BurstQPlan &qp, const QualAcc *part, uint32_t nt)
{
    const BurstItem &x = p.items[it];
    QualAcc q = x.q;
    if (qp.run) {
        qual_zero(q);
        for (uint32_t t = 0; t < nt; t++) qual_add(q, part[t]);
    }
    if (x.out >= 0) { p.qout[x.out] = q; return; }
    BurstDev &bd = *p.bd;
    bd.q = q; bd.qdone = (x.qdone || qp.run) ? 1u : 0u;
}

#ifndef WMB_HOSTSIM
__global__ void kb_mask_kernel(const BurstParams p)
{
    const uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi < WMB_BURST_LOOK + p.nw) kb_mask(p, wi);
}
__global__ void kb_count_kernel(const BurstParams p)
{
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u < p.units) p.cnt[u] = kb_events(p, u, false);
}
__global__ void kb_write_kernel(const BurstParams p)
{
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u < p.units) kb_events(p, u, true);
}
__global__ void __launch_bounds__(WMB_BURST_BLOCK) kb_runs_kernel(const BurstParams p)
{
    __shared__ BurstRunCtx r;
    __shared__ uint32_t cnt[WMB_BURST_BLOCK];
    __shared__ uint32_t total;
    if (threadIdx.x == 0) { kb_run_ctx(p, r); total = 0; }
    __syncthreads();
    const uint32_t chunks = (r.n_runs + WMB_BURST_BLOCK - 1) / WMB_BURST_BLOCK;
    for (uint32_t ch = 0; ch < chunks; ch++) {
        kb_runs_count(p, r, ch, threadIdx.x, cnt);
        __syncthreads();
        if (threadIdx.x == 0) kb_runs_scan(cnt, &total);
        __syncthreads();
        kb_runs_write(p, r, ch, threadIdx.x, cnt);
        __syncthreads();
    }
    if (threadIdx.x == 0) kb_runs_finish(p, r, total);
}
__global__ void __launch_bounds__(WMB_BURST_BLOCK) kb_reduce_kernel(const BurstParams p)
{
    __shared__ BurstPart part[WMB_BURST_BLOCK];
    __shared__ QualAcc qpart[WMB_BURST_BLOCK];
    __shared__ BurstQPlan qp;
    const uint32_t n = p.bd->n_items;
    for (uint32_t it = blockIdx.x; it < n; it += gridDim.x) {
        kb_reduce_part(p, it, threadIdx.x, WMB_BURST_BLOCK, part);
        __syncthreads();
        if (threadIdx.x == 0) kb_reduce_finish(p, it, part, WMB_BURST_BLOCK, p.qout ? &qp : nullptr);
        __syncthreads();
        if (p.qout) {                                   /* the launch's parameter: the whole block takes this branch */
            kb_qual_part(p, qp, threadIdx.x, WMB_BURST_BLOCK, qpart);
            __syncthreads();
            if (threadIdx.x == 0) kb_qual_finish(p, it, qp, qpart, WMB_BURST_BLOCK);
            __syncthreads();
        }
    }
}
#endif
