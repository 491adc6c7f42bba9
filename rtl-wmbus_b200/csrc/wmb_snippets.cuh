/*
 * wmb_snippets.cuh -- burst snippets (wmb_set_snippets / wmb_take_snippets, DESIGN.md §8): the raw cu8 bytes around
 * every burst piece, kept on the device before the batch's input buffer is reused.
 *
 * A granule is 2048 decimated samples (2048 d IQ samples, 4096 d bytes).  The snippet of a piece [s, e) covers the
 * granules [floor(s / 2048) - PRE, ceil(e / 2048) + POST).  Per batch, on cs in the gather that runs the burst pass,
 * behind kb_mask:
 *   ksn_keep   thread per granule g of the batch: keep[g] = 1 when an above sample of a burst-on chain lies in the
 *              granules [g - POST - 1, g + PRE + 1].  Above samples of earlier batches enter through SnipDev.la1 (the
 *              last granule with one); the batch's last PRE + 1 granules are always kept, because whether the next
 *              batch starts a piece within PRE granules of them is not known yet, and their bytes will be gone then.
 *   (count scan of keep -> each kept granule's rank, and their number)
 *   ksn_copy   block per granule: a kept one writes its batch index to the slot's list and, when its rank fits the
 *              slot's pool, its bytes to the pool (16-byte loads).
 * Why that keeps every granule of every snippet (the keep lemma): a piece's first sample s is an above sample or a cut,
 * its last sample e - 1 is an above sample or lies before a cut, and inside a run every sample lies within G <= 196 <
 * 2048 samples of an above sample, whether the piece is open, cut or bridged.  So every granule in [floor(s / 2048),
 * ceil(e / 2048)) is within one granule of a granule with an above sample of the piece, the PRE granules before it are
 * within PRE + 1 of one, the POST granules after it within POST + 1.
 */
#pragma once

#define WMB_SNIP_GRAN   2048               /* decimated samples per granule                                  */
#define WMB_SNIP_PRE    WMB_SNIPPET_PRE    /* granules kept before a piece's first granule (include/wmbus_b200.h) */
#define WMB_SNIP_POST   WMB_SNIPPET_POST   /* granules kept after its last one */
#define WMB_SNIP_BLOCK  256u               /* threads of ksn_keep / ksn_copy                                 */
#define WMB_SNIP_POOL_MAX (64ull << 20)    /* bytes of a result slot's pool at most                          */

struct SnipDev {                    /* carried from batch to batch */
    uint64_t la1;                   /* 1 + the last absolute granule with an above sample before this batch (0: none) */
    uint64_t la1_next;              /* ... including this batch (ksn_keep raises it, ksn_copy moves it to la1)          */
};

struct SnipParams {
    const uint32_t *mask[WMB_N_CHAINS];  /* kb_mask words of the burst-on chains (null: off), [WMB_BURST_LOOK + nw]  */
    uint32_t nw;                    /* mask words of the batch                                                     */
    uint32_t ng;                    /* granules of the batch (the last may be partial at the end of input)       */
    uint64_t g0;                    /* absolute granule of batch sample 0                                          */
    uint32_t *keep;                 /* [ng]                                                                        */
    const uint64_t *rank;           /* [ng], the count scan of keep                                                */
    SnipDev *sd;
    const uint8_t *in;              /* the batch's cu8 bytes                                                       */
    uint64_t in_bytes;
    uint32_t gbytes;                /* 4096 d                                                                      */
    uint32_t pool_gran;             /* granules the slot's pool holds                                              */
    uint8_t *pool;                  /* this slot's pool                                                            */
    uint32_t *list;                 /* this slot's kept granules (batch indices), in order                        */
};

/* the granule holds an above sample of a burst-on chain: its 64 mask words (fewer for a partial last granule) */
WMB_D bool ksn_any(const SnipParams &p, int64_t g)
{
    if (g < 0 || g >= (int64_t)p.ng) return false;
    const uint32_t w0 = (uint32_t)g * (WMB_SNIP_GRAN / 32), w1 = w0 + WMB_SNIP_GRAN / 32 < p.nw ? w0 + WMB_SNIP_GRAN / 32 : p.nw;
    uint32_t acc = 0;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!p.mask[ch]) continue;
        for (uint32_t w = w0; w < w1; w++) acc |= p.mask[ch][WMB_BURST_LOOK + w];
    }
    return acc != 0;
}

/* any[] over the batch granules [b0 - POST - 1, b0 + n + PRE + 1), entry i for granule b0 - POST - 1 + i */
#define WMB_SNIP_HALO (WMB_SNIP_PRE + WMB_SNIP_POST + 2)
WMB_D void ksn_keep_fill(const SnipParams &p, uint32_t b0, uint32_t i, uint8_t *any)
{
    const int64_t g = (int64_t)b0 - (WMB_SNIP_POST + 1) + (int64_t)i;
    const bool a = ksn_any(p, g);
    any[i] = a ? 1 : 0;
    if (a && i >= WMB_SNIP_POST + 1 && i < WMB_SNIP_POST + 1 + WMB_SNIP_BLOCK) {
#ifdef WMB_HOSTSIM
        if (p.sd->la1_next < p.g0 + (uint64_t)g + 1) p.sd->la1_next = p.g0 + (uint64_t)g + 1;
#else
        atomicMax((unsigned long long *)&p.sd->la1_next, (unsigned long long)(p.g0 + (uint64_t)g + 1));
#endif
    }
}
WMB_D void ksn_keep_decide(const SnipParams &p, uint32_t b0, uint32_t t, const uint8_t *any)
{
    const uint32_t g = b0 + t;
    if (g >= p.ng) return;
    bool k = g + (WMB_SNIP_PRE + 1) >= p.ng;                          /* decided by the next batch */
    /* an above sample of an earlier batch within POST + 1 granules before g */
    if (p.sd->la1 && p.sd->la1 - 1 + (WMB_SNIP_POST + 1) >= p.g0 + g) k = true;
    for (uint32_t i = t; i <= t + WMB_SNIP_PRE + WMB_SNIP_POST + 2; i++) k = k || any[i];
    p.keep[g] = k ? 1u : 0u;
}

/* ksn_copy, thread t of nt for granule g */
WMB_D void ksn_copy_part(const SnipParams &p, uint32_t g, uint32_t t, uint32_t nt)
{
    if (!p.keep[g]) return;
    const uint64_t k = p.rank[g];
    if (t == 0) p.list[k] = g;
    if (k >= p.pool_gran) return;                                     /* lost: the host marks it */
    const uint64_t at = (uint64_t)g * p.gbytes;
    const uint64_t n = (at + p.gbytes <= p.in_bytes ? p.gbytes : p.in_bytes - at) / 16;   /* the input is in 4096-byte items */
#ifdef WMB_HOSTSIM
    if (t == 0) memcpy(p.pool + k * p.gbytes, p.in + at, (size_t)n * 16);
    (void)nt;
#else
    const uint4 *src = (const uint4 *)(p.in + at);
    uint4 *dst = (uint4 *)(p.pool + k * p.gbytes);
    for (uint64_t i = t; i < n; i += nt) dst[i] = src[i];
#endif
}

#ifndef WMB_HOSTSIM
__global__ void __launch_bounds__(WMB_SNIP_BLOCK) ksn_keep_kernel(const SnipParams p)
{
    __shared__ uint8_t any[WMB_SNIP_BLOCK + WMB_SNIP_HALO];
    const uint32_t b0 = blockIdx.x * WMB_SNIP_BLOCK;
    for (uint32_t i = threadIdx.x; i < WMB_SNIP_BLOCK + WMB_SNIP_HALO; i += WMB_SNIP_BLOCK) ksn_keep_fill(p, b0, i, any);
    __syncthreads();
    ksn_keep_decide(p, b0, threadIdx.x, any);
}
__global__ void __launch_bounds__(WMB_SNIP_BLOCK) ksn_copy_kernel(const SnipParams p)
{
    /* ksn_keep is done with la1: the next batch sees this one's above samples */
    if (blockIdx.x == 0 && threadIdx.x == 0) p.sd->la1 = p.sd->la1_next;
    ksn_copy_part(p, blockIdx.x, threadIdx.x, WMB_SNIP_BLOCK);
}
#endif
