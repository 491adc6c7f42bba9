/*
 * wmb_context.cu -- host side of libwmbus_b200.so: the C ABI declared in
 * include/wmbus_b200.h, device buffers, stream orchestration and the stream/batch
 * bookkeeping around the kernels in wmb_kernels.cuh.
 *
 * Per batch of IQ bytes (stream-ordered on the context's compute stream):
 *     H2D (copy stream, double-buffered)                       [host input only]
 *     K1  k1_demod_kernel        cu8 -> dphi (fp32) + rssi (u8), both chains
 *     K2a k2a_lanes_kernel       clock recovery lanes -> packed data bits + time2 strobes
 *         k2a_verify_kernel      compare lane start states with predecessors' end states;
 *                                refuted lanes are re-run until none is left
 *     K2t count / scan / write   time2 bit stream -> stream ring, access-code matches
 *     K2m k2m_lanes_kernel       run-length lanes (+ verify / re-run)
 *     K2c scan + compact         run-length events -> stream ring, access-code matches
 *     K3  size/offsets/copy      candidate frames -> pinned host memory
 * The host then owns 3-out-of-6 / Manchester / CRC (wmb_framer.c), exactly the split
 * BASELINE.json's north_star asks for.
 *
 * With -DWMB_HOSTSIM the same file builds against tests/hostsim/hostsim_cuda.h and runs
 * the kernels' phase functions on the CPU; that build is test infrastructure only.
 */
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>
#include <thread>
#include <time.h>

#ifdef WMB_HOSTSIM
#include "hostsim_cuda.h"
#else
#include <cuda_runtime.h>
#endif

#include "wmbus_b200.h"
#include "wmb_framer.h"
#include "wmb_kernels.cuh"
#include "wmb_bursts.cuh"
#include "wmb_snippets.cuh"
#include "wmb_spectrum.cuh"

#ifndef WMB_VERSION
#define WMB_VERSION "wmbus-b200 0.1 (sm_90a)"
#endif

static thread_local char g_err[512];

static int set_err(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess)                                                                 \
            return set_err(WMB_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                                \
    } while (0)

/* --------------------------------------------------------------------------- */

struct Stream {                     /* one (chain, algo) bit stream */
    uint32_t *ev = nullptr;         /* run-length: lane-local events              */
    uint32_t *cnt = nullptr;        /* per-lane (time2: per-tile) counts          */
    uint64_t *base = nullptr;       /* per-lane (time2: per-tile) ordinal base    */
    uint64_t *ring = nullptr;       /* global event ring                          */
    uint64_t ring_cap = 0;          /* power of two                               */
    StreamDev *sd = nullptr;        /* device bookkeeping                         */
    uint64_t *cand = nullptr;       /* device: new access-code matches (ordinals, unordered) */
    uint64_t *pend = nullptr;       /* device: candidates waiting for more bits   */
    OfsAcc *pend_ofs = nullptr;     /* device: their carrier-offset sums          */
    QualAcc *pend_qual = nullptr;   /* device: their quality sums (quality on)    */
    int16_t *soft_ring = nullptr;   /* device: soft values beside ring (soft values on; S1: its values on) */
    uint64_t *agg = nullptr;        /* scan scratch [tiles]                       */
    uint64_t total = 0;             /* host mirror of sd->total at the last read  */
    uint64_t total_prev = 0;        /* ... before the last batch read (stage tap) */
    /* host framer bookkeeping */
    int64_t busy_until = -1;        /* last ordinal consumed by an accepted packet */
    std::vector<uint64_t> rep_wait; /* repair on: accepted S1 aborts booked while partial, waiting for bit P - 1 (ordinals, ascending) */
};

/* Buffers that the demod / clock-recovery stage of batch i+1 writes while the bit-stream stage of batch i still
 * reads them: two sets, alternating from batch to batch.  Layout of the sample arrays: [W history | batch]. */
struct SetBuf {
    float *dphi = nullptr;          /* [W | M_max]  post-FIR discriminator output  */
    uint8_t *rssi = nullptr;        /* [W | M_max]                                 */
    uint32_t *dbits = nullptr;      /* [W/32 | M_max/32] data bits                 */
    uint32_t *sbits = nullptr;      /* [W/32 | M_max/32] time2 strobes             */
    uint32_t *cbits = nullptr;      /* [W/32 | M_max/32] clock signs (stage tap, opts.reserved[1] & 1) */
    IirState *ia_start = nullptr, *ia_end = nullptr;
    uint32_t *rerun_a = nullptr;
};

struct ChainBuf {
    SetBuf set[2];
    IirState *ia_carry = nullptr;
    RlState *rl_start = nullptr, *rl_end = nullptr, *rl_carry = nullptr;
    uint32_t *rerun = nullptr;
    uint32_t *lane_err = nullptr;   /* [lanes_max] error bits of the run-length lanes' verified runs */
    /* two-phase run-length path (T1/C1) */
    uint64_t *p1_rec = nullptr; uint32_t *p1_cnt = nullptr; uint64_t *p1_base = nullptr;
    P1State *p1_start = nullptr, *p1_end = nullptr; uint32_t *p1_rerun = nullptr;
    uint32_t *rec_m = nullptr, *rec_v = nullptr; uint16_t *rec_n = nullptr;
    uint32_t *p2_cnt = nullptr; uint64_t *p2_base = nullptr;
    K2pDev *pd = nullptr; RlState *p2_out = nullptr;
    /* time2 tiles */
    uint32_t *t2_tail = nullptr, *t2_len = nullptr, *t2_sr = nullptr, *t2_agg_tail = nullptr, *t2_agg_len = nullptr;
    Stream s[WMB_N_ALGOS];
};

#define WMB_NSLOT 4                      /* batches whose results may be waiting for the host */

/* One kind of per-batch result: a device array of WMB_NSLOT x parts x cap elements and its pinned host mirror.  The
 * copy enqueued behind a gather fetches a prefix of each (slot, part), since the host cannot know yet how many elements
 * the batch wrote.  Once the count has been read the host fetches the rest and grows the prefix so that later batches
 * fit it.  Several gathers are in flight at once, so the rest of a slot starts at what that slot's own copy fetched
 * (wmb_ctx::InFlight), never at the current prefix, which may have grown since. */
template <typename T> struct SlotTable {
    T *d = nullptr, *h = nullptr;
    size_t cap = 0;                 /* elements per slot and part */
    uint32_t parts = 1;
    uint32_t prefix = 0;            /* elements the next prefix copy fetches */
    uint32_t slack = 0;             /* growth beyond n + n / 4 */

    size_t at(int slot, int part = 0) const { return ((size_t)slot * parts + part) * cap; }
    int alloc(wmb_ctx *c, uint32_t n_parts, size_t n_cap, uint32_t first_prefix, uint32_t grow_slack);
    int release(wmb_ctx *c);
    /* elements [copied, n) of (slot, part) on st when n > copied; sets *issued (if given) when it copies */
    int fetch(int slot, int part, uint32_t copied, uint32_t n, cudaStream_t st, bool *issued = nullptr) const
    {
        if (n <= copied) return WMB_OK;
        if (n > cap) return set_err(WMB_E_STATE, "internal: batch results beyond their slot table");
        const size_t i = at(slot, part) + copied;
        CUDA_TRY(cudaMemcpyAsync(h + i, d + i, (size_t)(n - copied) * sizeof(T), cudaMemcpyDeviceToHost, st));
        if (issued) *issued = true;
        return WMB_OK;
    }
    /* the prefix copy of (slot, part) on st; *copied: the elements it fetches */
    int enqueue(int slot, int part, cudaStream_t st, uint32_t *copied) const { *copied = prefix; return fetch(slot, part, 0, prefix, st); }
    void grow(uint32_t n) { if (n > prefix) prefix = (uint32_t)std::min<size_t>(cap, (size_t)n + n / 4 + slack); }
};

static uint32_t g_p2_block = 128u;       /* threads per block of the phase-2 count pass (WMBUS_B200_P2BLK, experiments) */

struct QueuedLine {
    uint64_t end_sample;
    int prio;                       /* chain*2 + (algo == T2A) */
    wmb_decoded d;
    uint8_t algo, chain;
    uint8_t ofs_valid;              /* 0: the frame came from the caller (wmb_decode_frames), no sum */
    uint64_t sync_sample;           /* access-code match */
    int64_t ofs_sum;                /* carrier-offset window (FrameHdr) */
    uint32_t ofs_n;
    QualAcc qual;                   /* quality class sums (zero when the report is off or the frame came from the caller) */
};

/* a closed burst piece and its quality sums (wmb_take_bursts_quality) */
struct QueuedBurst {
    wmb_burst b;
    QualAcc q;
};

struct wmb_ctx {
    wmb_opts o;
    int device = 0;
    uint32_t d = 2;                 /* effective decimation (>= 1) */
    uint32_t chains = 3;
    /* Streams: k1s runs the demod kernels of consecutive batches back to back; as[set] the clock-recovery lanes of
     * a batch (they only need its demod output, so they overlap the next batch's demod and each other); cs everything
     * that is sequential from batch to batch (lane verification, bit streams, gather, framer, result copies), with ts
     * (time2) and s2 (S1 run-length lanes) forked from and joined to it; xs the H2D copies.  When the demod kernel
     * slices the data bits, the run-length path starts behind it instead, beside the clock lanes: T1/C1 on rs, S1 on
     * s2, both forked from cs at the start of the batch (run_batch). */
    cudaStream_t cs = nullptr, xs = nullptr, k1s = nullptr, as[2] = {nullptr, nullptr}, as2[2] = {nullptr, nullptr};
    cudaStream_t ts = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaStream_t s2 = nullptr;
    cudaEvent_t ev_fork2 = nullptr, ev_join2 = nullptr;
    cudaStream_t rs = nullptr;
    cudaEvent_t ev_join_rs = nullptr;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_k1done[2] = {nullptr, nullptr};
    cudaEvent_t ev_k1[2] = {nullptr, nullptr}, ev_k2a[2] = {nullptr, nullptr}, ev_k2a2[2] = {nullptr, nullptr}, ev_chain[2] = {nullptr, nullptr};
    bool chain_recorded[2] = {false, false};
    cudaEvent_t ev_res[WMB_NSLOT] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_push_start = nullptr;           /* first demod kernel of the current push (timers) */
    cudaEvent_t ev_reset = nullptr;                /* wmb_reset's device part (the first batch after it waits for it) */
    bool reset_pending = false;
    bool push_started = false;
    cudaEvent_t ev_t[WMB_NSLOT][6];                /* per result slot: demod start/end, bit sync start/end (timers) */
    bool allocated = false;

    /* geometry */
    size_t max_batch_bytes = 0;
    int64_t M_max = 0;
    uint32_t W = 32768;             /* retained history (decimated samples) = max warm-up */
    uint32_t W_a[WMB_N_CHAINS] = {24576, 81920};    /* warm-up of the clock-recovery lanes */
    uint32_t W_m[WMB_N_CHAINS] = {32768, 8192};    /* warm-up of the run-length lanes  */
    uint32_t C_fixed = 0;
    uint32_t lanes_max = 0;
    uint32_t t2_tiles_max = 0;
    uint32_t p1_lanes_max = 0, p2_lanes_max = 0;
    size_t rec_max = 0;
    bool two_phase = true;
    bool taps = false;              /* opts.reserved[1] & 1: keep the clock-sign words for wmb_debug_copy_bits */
    K2pDev *h_pd = nullptr;
    uint32_t cap_words_rl = 0;
    size_t ring_events = 0, ring_events_rl = 0;
    std::vector<void *> dev_allocs, host_allocs;
    uint8_t *d_tmp = nullptr;       /* scratch for the history slides                    */
    uint32_t cand_cap = 1u << 20;
    uint32_t frame_words_cap = 1u << 24;

    /* device buffers */
    uint8_t *d_in[2] = {nullptr, nullptr};
    uint8_t *d_hist = nullptr;
    float *d_lut = nullptr;
    ChainBuf cb[WMB_N_CHAINS];
    uint32_t *d_errors = nullptr, *d_nfail = nullptr;      /* [0] error bits; d_nfail[0..7]: refuted lanes per verified pass */
    GatherDev *d_gd = nullptr;      /* gather bookkeeping + statistics                 */
    /* results: WMB_NSLOT slots, one per batch in flight, each with its part of the candidate / verdict arrays and of
     * the datagram pool; the host mirrors are pinned and filled by copies enqueued right behind the device framer */
    BatchRec *d_rec = nullptr, *h_rec = nullptr;
    SlotTable<FrameHdr> hdr;
    SlotTable<DecHdr> dec;
    SlotTable<uint8_t> pool;
    uint32_t pend_cap = 0;
    uint32_t *d_words = nullptr, *h_words = nullptr;
    uint32_t *d_cut_n = nullptr;
    uint64_t *d_k3_agg = nullptr;
    /* a gathered batch; per table, the elements its prefix copy fetched (0: the table was not copied) */
    struct InFlight { int slot; bool final; bool has_timers; uint64_t m_end;
                      uint32_t hdr, dec, qual, pool, brec, bqual, ssum, speak, rep;
                      bool sn; uint64_t sn_g0, sn_bytes; uint32_t snlist, snpool;     /* the batch's kept granules */
                      uint64_t iq_end; };
    std::vector<InFlight> inflight;                  /* gathered batches whose results the host has not read yet */
    uint64_t stat_rerun_seen = 0, stat_fallback_seen = 0;
    double acc_demod_ms = 0, acc_bitsync_ms = 0, acc_pass_ms = 0;    /* timers of the current push */

    /* stream position */
    uint64_t iq_consumed = 0;       /* input IQ samples handed to the device    */
    uint64_t m_consumed = 0;        /* decimated samples produced               */
    int64_t hist_m = 0;             /* decimated history retained (<= W)        */
    int64_t hist_iq = 0;            /* input history retained (samples)         */
    std::vector<uint8_t> remainder; /* bytes not yet forming a whole batch granule */
    int buf_idx = 0;
    uint64_t batch_no = 0;          /* batches enqueued since create / reset: set = batch_no & 1 */
    uint64_t gather_no = 0;         /* gathers enqueued: result slot = gather_no % WMB_NSLOT    */
    int64_t last_M = 0, prev_M = 0;
    int64_t last_hist = 0;          /* samples before the last batch's first one that exist since reset / seek (<= W) */
    int last_set = 0;
    double fir_gain[WMB_N_CHAINS] = {1.0, 1.0};     /* DC gain of each chain's post-demod FIR (wmb_line_info.offset_hz) */

    /* receiver settings per chain (wmb_set_receiver; they survive wmb_reset) */
    uint32_t lock[WMB_N_CHAINS] = {2, 2};            /* clock-lock threshold, rtl_wmbus.c:865-866 */
    uint32_t ac_err[WMB_N_CHAINS] = {0, 0};          /* access-code bit errors, :99, :103         */

    /* burst report (wmb_set_bursts; the levels survive wmb_reset).  Level 0: off, nothing is allocated or launched */
    uint32_t burst_level[WMB_N_CHAINS] = {0, 0};
    struct BurstBuf { uint32_t *mask = nullptr, *cnt = nullptr; uint64_t *base = nullptr, *agg = nullptr; int64_t *ev = nullptr;
                      BurstDev *bd = nullptr; BurstItem *items = nullptr; } bb[WMB_N_CHAINS];
    bool burst_allocated = false;
    SlotTable<BurstRec> brec;                        /* [WMB_NSLOT][chain][cap] */
    BurstSlot *d_bslot = nullptr, *h_bslot = nullptr;
    std::vector<QueuedBurst> bursts;                 /* closed pieces not taken yet */
    uint64_t burst_frontier = 0;                     /* no piece still to come starts before this sample */

    /* burst snippets (wmb_set_snippets; the mode survives wmb_reset).  0: off, nothing is allocated, launched or copied */
    uint32_t snip_mode = 0;
    uint32_t *d_snkeep = nullptr;
    uint64_t *d_snrank = nullptr, *d_snagg = nullptr;
    SnipDev *d_snd = nullptr;
    uint64_t *d_snn = nullptr, *h_snn = nullptr;     /* [WMB_NSLOT] granules the slot's batch kept */
    uint32_t snip_pool_gran = 0;                     /* granules a slot's pool holds */
    SlotTable<uint32_t> snlist;                      /* [WMB_NSLOT][granules of a batch]: the kept ones, in order */
    SlotTable<uint8_t> snpool;                       /* [WMB_NSLOT][snip_pool_gran * 4096 d]: their bytes */
    cudaEvent_t ev_snip[2] = {nullptr, nullptr};     /* ksn_copy is done with d_in[i] */
    const uint8_t *last_src = nullptr;               /* the last batch's input bytes (d_in[i] or the caller's) */
    size_t last_bytes = 0;
    struct SnipGran { std::vector<uint8_t> bytes; bool lost; };
    std::map<uint64_t, SnipGran> sn_store;           /* kept granules by absolute index */
    std::vector<wmb_snippet> sn_queue;               /* burst pieces whose snippets are not handed out yet */
    std::set<uint64_t> sn_ok[WMB_N_CHAINS];          /* access-code matches of CRC-ok lines and repaired telegrams */
    uint64_t sn_iq_end = 0;                          /* input consumed by the batches booked so far (IQ samples) */
    uint64_t sn_g_first = 0;                         /* first granule pushed since wmb_reset / wmb_seek */

    /* telegrams (wmb_set_telegrams; survives wmb_reset).  Off: nothing is kept */
    bool telegrams = false;
    std::vector<wmb_line_info> tg_info;              /* the lines and REPAIRED records of groups not final yet */
    std::vector<wmb_decoded> tg_line;                /* parallel to tg_info */
    std::vector<wmb_repair_record> tg_rep;
    struct ReadyTelegram { wmb_telegram t; std::vector<uint8_t> bytes; };
    std::vector<ReadyTelegram> tg_ready;             /* records of final groups not handed out yet, in order */

    bool flushed = false;                            /* the end-of-input gather has been booked (snippets, telegrams) */

    /* signal quality (wmb_set_line_quality; survives wmb_reset).  Off: nothing is allocated, launched or copied */
    bool quality = false;
    SlotTable<QualAcc> qual;                        /* parallel to hdr */
    SlotTable<QualAcc> bqual;                        /* parallel to brec */

    /* erasure repair of the framer's candidates (wmb_set_repair; survives wmb_reset).  0: off, nothing is allocated,
     * launched or copied */
    uint32_t repair_e = 0;
    SlotTable<RepHdr> rep;                           /* parallel to hdr */
    std::vector<wmb_repair_record> repairs;          /* records not taken yet */

    /* soft values of the T1/C1 bits (wmb_set_soft_bits on a manual_frames context, or the streaming soft repair; both survive
     * wmb_reset).  Off: nothing is allocated or launched */
    bool soft = false;
    uint32_t repair_k = 0;                           /* wmb_set_repair_soft: k_max of the C1 soft repair K4S (0: off) */
    uint32_t repair_s = 0;                           /* wmb_set_repair_t1_soft: s_max of the T1 soft repair K4S (0: off) */
    bool soft_s1 = false;                            /* wmb_set_soft_bits_s1 (manual_frames): S1 soft values too */
    uint32_t repair_s1 = 0;                          /* wmb_set_repair_s1_soft: s_max of the S1 soft repair K4S (0: off) */
    int16_t *d_soft_words = nullptr, *h_soft_words = nullptr;    /* parallel to d_words / h_words */

    /* band survey (wmb_set_spectrum; the setting survives wmb_reset).  Bins 0: off, nothing is allocated or launched */
    uint32_t spec_bins = 0, spec_B = 0;
    uint32_t spec_R = 0;                             /* ring rows = rows of a result slot: batch blocks / B + 2 */
    uint32_t spec_tab_n = 0;                         /* N of the tables on the device */
    float *d_spec_tab = nullptr;                     /* hann[N] | tw[N / 2][2] */
    uint64_t *d_ssum_ring = nullptr;                 /* [R][N] */
    uint32_t *d_speak_ring = nullptr;
    SlotTable<uint64_t> ssum;                        /* [WMB_NSLOT][R][N] */
    SlotTable<uint32_t> speak;
    cudaEvent_t ev_spec = nullptr;                   /* the batch's survey kernels are done (cs waits before its copies) */
    cudaEvent_t ev_spec_flush = nullptr;             /* the flush's close is done (the next batch's survey waits) */
    bool spec_flush_pending = false;
    bool spec_enqueued = false;                      /* a batch's survey kernels are on the demod stream, cs not yet behind them */
    int64_t spec_open = -1;                          /* record of the last block pushed, while it has blocks counted */
    uint32_t spec_open_blocks = 0;
    std::vector<wmb_spectrum_row> spec_batch_rows;   /* rows the last batch closed, until its gather takes them */
    std::vector<wmb_spectrum_row> spec_slot_rows[WMB_NSLOT];
    std::vector<wmb_spectrum_row> spec_rows;         /* closed records not taken yet, with their bins */
    std::vector<uint64_t> spec_sum;
    std::vector<uint32_t> spec_peak;

    /* results */
    uint64_t win_lo = 0, win_hi = ~0ull;             /* line window (access-code match sample) */
    /* manual mode (opts.manual_frames): frames wait here for wmb_poll */
    struct Held { wmb_frame f; std::vector<uint32_t> words; std::vector<int16_t> soft; /* empty: none */ };
    std::vector<Held> held, held_prev;
    std::vector<wmb_frame> poll_frames;
    bool manual = false;
    std::vector<QueuedLine> lines;
    wmb_stats st;
};

/* --------------------------------------------------------------------------- */
/* launches                                                                    */
/* --------------------------------------------------------------------------- */

static uint32_t *gd_field(wmb_ctx *c, size_t off) { return (uint32_t *)((uint8_t *)c->d_gd + off); }
#define GD_FIELD(c, f) gd_field(c, offsetof(GatherDev, f))

#ifdef WMB_HOSTSIM
#include "hostsim_launch.inl"
/* The demod kernel's wide tile (k1_rows_per_thread(): d = 1 or the d = 2 fast path, so neither the prefilter nor the
 * separate box / discriminator phases occur) in the CPU build, with the narrow tile's structure: each barrier-separated
 * phase over all producer threads, then the RSSI warp's lanes.  Narrow tiles go through launch_k1 of hostsim_launch.inl. */
template <class CH>
static void hostsim_k1_wide_chain(const K1Params &p, K1Smem &sm, const uint8_t *raw, int64_t tile, bool need_convert)
{
    const bool fast = p.d == 2u;
    if (need_convert) hs_for(K1_THREADS, [&](uint32_t t) {
        if (fast) k1_convert_fast(p, sm, raw, tile, t); else k1_convert<CH::ID>(p, sm, raw, tile, t);
    });
    if (fast) hs_for(K1_THREADS, [&](uint32_t t) { k1_box_disc<CH, 1, true, K1_RPT_WIDE>(p, sm, t); });
    else hs_for(K1_THREADS, [&](uint32_t t) { k1_box_disc<CH, 1, false, K1_RPT_WIDE>(p, sm, t); });
    hs_for(K1_THREADS, [&](uint32_t t) { k1_fir<CH, K1_RPT_WIDE>(p, sm, tile, t); });
    hs_for(32, [&](uint32_t t) { k1_rssi<CH, K1_RPT_WIDE>(p, sm.mag, tile, t); });      /* the block's RSSI warp */
}

static int launch_demod(wmb_ctx *c, const K1Params &p, cudaStream_t st)
{
    if (p.rpt != K1_RPT_WIDE) return launch_k1(c, p, st);
    const int64_t ntiles = (p.M + K1Geo<K1_RPT_WIDE>::TILE - 1) / K1Geo<K1_RPT_WIDE>::TILE;
    std::vector<uint8_t> smem(k1_smem_bytes(p.d, p.prefilter, p.rpt) + 256, 0xA5);   /* garbage-filled like real smem */
    K1Smem sm;
    uint8_t *base = smem.data();
    base += (128 - ((uintptr_t)base & 127)) & 127;
    k1_carve(sm, base, p.d, p.prefilter, p.rpt);
    hs_for(WMB_ATAN_TAB_ELEMS, [&](uint32_t i) { wmb_atan_tab_fill((WmbAtanTab *)base, i); });
    int rc = WMB_OK;
    hs_for((uint32_t)ntiles, [&](uint32_t tile) {
        const K1Load L = k1_plan_load(p, tile);
        if (L.n0) memcpy(sm.bytes[0], L.src0, (size_t)L.n0);
        if (L.n1) memcpy(sm.bytes[0] + L.off1, L.src1, (size_t)L.n1);
        if ((L.n0 | L.n1 | L.off1) & 15) { rc = set_err(WMB_E_STATE, "hostsim: unaligned bulk copy"); return; }
        const uint8_t *raw = sm.bytes[0];
        if (p.chains & 1u) hostsim_k1_wide_chain<ChainT1C1>(p, sm, raw, tile, true);
        if (p.chains & 2u) hostsim_k1_wide_chain<ChainS1>(p, sm, raw, tile, p.mix || !(p.chains & 1u));
    });
    c->st.kernel_launches++;
    return rc;
}
/* the CPU build runs every launch when it is enqueued, in the order of the calls: the stream is not needed */
static int launch_k2p1(wmb_ctx *c, const K2p1Params &p, cudaStream_t) { return launch_k2p1(c, p); }
static int launch_k2p_rest(wmb_ctx *c, const K2pcParams &pc, const K2p2Params &p2, cudaStream_t) { return launch_k2p_rest(c, pc, p2); }
static int launch_k2p_fold(wmb_ctx *c, const P1State *p1_end_last, RlState *p2_out, RlState *carry, const K2pDev *pd,
                           const RlState *mono_end, cudaStream_t)
{
    return launch_k2p_fold(c, p1_end_last, p2_out, carry, pd, mono_end);
}
/* the gather with the erasure repair K4R (r given): on the device K4R runs between K4 and k3_publish, which reads the
 * pool_n that K4R adds to.  Here the simulated gather has published already, so K4R runs behind it and the batch is
 * published again, with the capacity flags the first publish cleared (n_pend's clamp is idempotent): the record is the
 * one the device writes */
static int launch_k3_k4(wmb_ctx *c, const K3Params &p, const K4Params *q, const K4RParams *r, const K4SParams *sp)
{
    const int rc = launch_k3_k4(c, p, q);
    if (rc) return rc;
    /* soft values: on the device k3_soft runs between k3_cut and k3_copy.  It reads only what k3_size and k3_cut wrote
     * (cut_n, never changed again), so here it runs behind the simulated gather, and the copy is redone (the frame words
     * it writes are the same again) */
    if (p.soft_words) {
        const uint32_t n = p.gd->n;
        hs_for(n, [&](uint32_t i) { hs_for(4, [&](uint32_t t) { k3_soft<false>(p, i, t, 4); }); });
        c->st.kernel_launches += 1;
        if (p.soft_ring[WMB_CHAIN_S1 * WMB_N_ALGOS + WMB_ALGO_RLA] || p.soft_ring[WMB_CHAIN_S1 * WMB_N_ALGOS + WMB_ALGO_T2A]) {
            hs_for(n, [&](uint32_t i) { hs_for(4, [&](uint32_t t) { k3_soft<true>(p, i, t, 4); }); });
            c->st.kernel_launches += 1;
        }
        hs_for(n, [&](uint32_t i) { hs_for(4, [&](uint32_t t) { k3_copy(p, i, t, 4); }); });
    }
    if (!r) return WMB_OK;
    static K4RSmem sm;                  /* the block's phases need real barriers: one simulated thread */
    hs_for(p.gd->n, [&](uint32_t i) { k4r_repair(*r, i, 0, 1, sm); });
    c->st.kernel_launches += 1;
    if (sp) {
        static K4SSmem ss;
        if (sp->k_max || sp->s_max) {
            hs_for(p.gd->n, [&](uint32_t i) { k4s_repair<false>(*sp, i, 0, 1, ss); });
            c->st.kernel_launches += 1;
        }
        if (sp->s1_max) {
            hs_for(p.gd->n, [&](uint32_t i) { k4s_repair<true>(*sp, i, 0, 1, ss); });
            c->st.kernel_launches += 1;
        }
    }
    *p.errors |= p.rec->errors & K3_SOFT_ERRORS;
    k3_publish(p);
    return WMB_OK;
}
#else
static int g_k1_ctas = 0;                /* WMBUS_B200_K1_CTAS: resident demod blocks per SM (0: as many as fit) */

static int launch_demod(wmb_ctx *c, const K1Params &p, cudaStream_t st)
{
    const int64_t tile = k1_tile_len(p.rpt);
    const int64_t ntiles = (p.M + tile - 1) / tile;
    /* `-p S -p T` turns both chains off: no chain buffer exists, and there is nothing to demodulate */
    if (ntiles <= 0 || p.chains == 0u) return WMB_OK;
    static int sm_count = 0, blocks_per_sm = 0;
    const size_t smem = k1_smem_bytes(p.d, p.prefilter, p.rpt);
    if (!sm_count) {
        cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, c->device);
    }
    const bool wide = p.rpt == K1_RPT_WIDE;
    auto kern = p.prefilter ? (p.chains == 1u ? k1_demod_pre_kernel<1u> : p.chains == 2u ? k1_demod_pre_kernel<2u> : k1_demod_pre_kernel<3u>)
              : wide ? (p.chains == 1u ? k1_demod_kernel<1u, K1_RPT_WIDE> : p.chains == 2u ? k1_demod_kernel<2u, K1_RPT_WIDE>
                                                                            : k1_demod_kernel<3u, K1_RPT_WIDE>)
                     : (p.chains == 1u ? k1_demod_kernel<1u, K1_RPT_NARROW> : p.chains == 2u ? k1_demod_kernel<2u, K1_RPT_NARROW>
                                                                              : k1_demod_kernel<3u, K1_RPT_NARROW>);
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kern, K1_BLOCK, smem));
    if (blocks_per_sm < 1) return set_err(WMB_E_INVAL, "decimation %u needs %zu B shared memory per CTA", p.d, smem);
    if (g_k1_ctas > 0 && blocks_per_sm > g_k1_ctas) blocks_per_sm = g_k1_ctas;
    int64_t grid = (int64_t)sm_count * blocks_per_sm;      /* persistent: whole waves of resident CTAs */
    if (grid > ntiles) grid = ntiles;
    CUDA_TRY(cudaMemsetAsync(p.tile_ctr, 0, 4, st));
    kern<<<(unsigned)grid, K1_BLOCK, smem, st>>>(p);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches++;
    return WMB_OK;
}

/* speculative pass (st: the batch's lane stream), then -- on cs, where batches follow each other in order --
 * verification + on-device fix-up of refuted lanes: no host round trip */
static int g_fixseg = 3;             /* WMBUS_B200_FIXSEG: parallel segment pass in front of the fix-up block for 1: clock lanes, 2: monolithic
                                            run-length lanes, 4: run-length phase 1 (off: its 2304-step lanes are cheap to re-run in one block, and the
                                            4096 idle blocks of the pass are pure overhead) */
static bool g_k2a_coop = true;           /* WMBUS_B200_K2A=scalar: one lane per thread everywhere (experiments) */

static int launch_k2a_lanes(wmb_ctx *c, int chain, const K2aParams &p, cudaStream_t st)
{
    /* three threads per lane where the lane is the plain case (time2 on, no DC block, whole words); the per-thread
     * kernel otherwise */
    if (g_k2a_coop && p.t2 && !p.dc && p.M % 32 == 0 && p.W % 32 == 0 && p.C % 32 == 0 && p.hist % 32 == 0) {
        const unsigned per = (K2A2_THREADS / 32) * K2A2_LPW;
        const unsigned grid = (p.lanes + per - 1) / per;
        if (p.lock == 2) {
            if (chain == 0) k2a2_lanes_kernel<ChainT1C1, 2><<<grid, K2A2_THREADS, 0, st>>>(p);
            else            k2a2_lanes_kernel<ChainS1, 2><<<grid, K2A2_THREADS, 0, st>>>(p);
        } else {
            if (chain == 0) k2a2_lanes_kernel<ChainT1C1, 0><<<grid, K2A2_THREADS, 0, st>>>(p);
            else            k2a2_lanes_kernel<ChainS1, 0><<<grid, K2A2_THREADS, 0, st>>>(p);
        }
        CUDA_TRY(cudaGetLastError());
        c->st.kernel_launches += 1;
        return WMB_OK;
    }
    const unsigned grid = (p.lanes + K2_THREADS - 1) / K2_THREADS;
    if (chain == 0) k2a_lanes_kernel<ChainT1C1><<<grid, K2_THREADS, 0, st>>>(p);
    else            k2a_lanes_kernel<ChainS1><<<grid, K2_THREADS, 0, st>>>(p);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 1;
    return WMB_OK;
}

static int launch_k2a_verify(wmb_ctx *c, int chain, const K2aParams &p)
{
    uint32_t *nf = c->d_nfail + chain;
    k2a_verify_kernel<<<(p.lanes + 255) / 256, 256, 0, c->cs>>>(p, nf);
    const unsigned segs = (p.lanes + FIX_SEG - 1) / FIX_SEG;
    if (chain == 0) {
        if (g_fixseg & 1) k2a_fixseg_kernel<ChainT1C1><<<segs, FIX_SEG, 0, c->cs>>>(p, nf, GD_FIELD(c, lanes_rerun));
        k2a_fixup_kernel<ChainT1C1><<<1, FIX_THREADS, 0, c->cs>>>(p, nf, GD_FIELD(c, lanes_rerun), c->d_errors);
    } else {
        if (g_fixseg & 1) k2a_fixseg_kernel<ChainS1><<<segs, FIX_SEG, 0, c->cs>>>(p, nf, GD_FIELD(c, lanes_rerun));
        k2a_fixup_kernel<ChainS1><<<1, FIX_THREADS, 0, c->cs>>>(p, nf, GD_FIELD(c, lanes_rerun), c->d_errors);
    }
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 3;
    return WMB_OK;
}

static int launch_k2m(wmb_ctx *c, int chain, const K2mParams &p, cudaStream_t st)
{
    const unsigned grid = (p.lanes + K2_THREADS - 1) / K2_THREADS;
    uint32_t *nf = c->d_nfail + 2 + chain;
    if (chain == 0) {
        k2m_lanes_kernel<ChainT1C1><<<grid, K2_THREADS, 0, st>>>(p);
        k2m_verify_kernel<<<(p.lanes + 255) / 256, 256, 0, st>>>(p, nf);
        if (g_fixseg & 2) k2m_fixseg_kernel<ChainT1C1><<<(p.lanes + FIX_SEG - 1) / FIX_SEG, FIX_SEG, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun));
        k2m_fixup_kernel<ChainT1C1><<<1, FIX_THREADS, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun), c->d_errors);
    } else {
        k2m_lanes_kernel<ChainS1><<<grid, K2_THREADS, 0, st>>>(p);
        k2m_verify_kernel<<<(p.lanes + 255) / 256, 256, 0, st>>>(p, nf);
        if (g_fixseg & 2) k2m_fixseg_kernel<ChainS1><<<(p.lanes + FIX_SEG - 1) / FIX_SEG, FIX_SEG, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun));
        k2m_fixup_kernel<ChainS1><<<1, FIX_THREADS, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun), c->d_errors);
    }
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 4;
    return WMB_OK;
}

static int launch_k2p1(wmb_ctx *c, const K2p1Params &p, cudaStream_t st)
{
    uint32_t *nf = c->d_nfail + 4;
    k2p1_lanes_kernel<<<(p.lanes + 127) / 128, 128, 0, st>>>(p);
    k2p1_verify_kernel<<<(p.lanes + 255) / 256, 256, 0, st>>>(p, nf);
    if (g_fixseg & 4) k2p1_fixseg_kernel<<<(p.lanes + FIX_SEG - 1) / FIX_SEG, FIX_SEG, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun));
    k2p1_fixup_kernel<<<1, FIX_THREADS, 0, st>>>(p, nf, GD_FIELD(c, lanes_rerun), c->d_errors);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 4;
    return WMB_OK;
}

static void launch_cscan(wmb_ctx *c, const uint32_t *cnt, uint64_t *base, uint32_t n, uint64_t *agg, uint64_t *total,
                         const uint32_t *skip = nullptr, uint32_t *clear = nullptr, uint32_t from_zero = 0, cudaStream_t st = nullptr,
                         uint32_t skip_invert = 0)
{
    if (!st) st = c->cs;
    CountScan s;
    s.cnt = cnt; s.base = base; s.n = n; s.agg = agg; s.total = total; s.skip = skip; s.clear = clear; s.from_zero = from_zero;
    s.skip_invert = skip_invert;
    const unsigned tiles = scan_tiles(n);
    cscan_a_kernel<<<tiles, SCAN_BLOCK, 0, st>>>(s);
    cscan_b_kernel<<<1, 32, 0, st>>>(s);
    cscan_c_kernel<<<tiles, SCAN_BLOCK, 0, st>>>(s);
    c->st.kernel_launches += 3;
}

/* two-phase run-length path after phase 1: records -> phase 2 -> ring (the carried state is folded later) */
static int launch_k2p_rest(wmb_ctx *c, const K2pcParams &pc, K2p2Params p2, cudaStream_t st)
{
    launch_cscan(c, pc.cnt, pc.base, pc.lanes, pc.agg, &pc.pd->n_rec, nullptr, &pc.pd->fallback, 1, st);
    k2pc_compact_kernel<<<pc.lanes, 128, 0, st>>>(pc);
    k2p2_count_kernel<<<(p2.lanes + g_p2_block - 1) / g_p2_block, g_p2_block, 0, st>>>(p2);
    k2p2_sum_kernel<<<p2.lanes, K2P2W_THREADS, 0, st>>>(p2);
    launch_cscan(c, p2.cnt, p2.base, p2.lanes, p2.agg, &p2.sd->total, &p2.pd->fallback, nullptr, 0, st);
    k2p2_write_kernel<<<p2.lanes, K2P2W_THREADS, 0, st>>>(p2);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 4;
    return WMB_OK;
}

static int launch_k2p_fold(wmb_ctx *c, const P1State *p1_end_last, RlState *p2_out, RlState *carry, const K2pDev *pd,
                           const RlState *mono_end, cudaStream_t st)
{
    k2p_fold_kernel<<<1, 32, 0, st>>>(p1_end_last, p2_out, carry, pd, mono_end, GD_FIELD(c, rl_fallbacks));
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 1;
    return WMB_OK;
}

static int launch_k2m_carry(wmb_ctx *c, const RlState *end, RlState *carry, const uint32_t *run_if, cudaStream_t st)
{
    k2m_carry_kernel<<<1, 32, 0, st>>>(end, carry, run_if);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 1;
    return WMB_OK;
}

static int launch_k2t(wmb_ctx *c, int chain, const K2tParams &p)
{
    const unsigned tiles = scan_tiles(p.lanes);
    if (chain == 0) {
        k2t_count_kernel<ChainT1C1><<<p.lanes, T2_THREADS, 0, c->ts>>>(p);
        t2scan_a_kernel<ChainT1C1><<<tiles, SCAN_BLOCK, 0, c->ts>>>(p);
        t2scan_b_kernel<ChainT1C1><<<1, 32, 0, c->ts>>>(p);
        t2scan_c_kernel<ChainT1C1><<<tiles, SCAN_BLOCK, 0, c->ts>>>(p);
        k2t_write_kernel<ChainT1C1><<<p.lanes, T2_THREADS, 0, c->ts>>>(p);
    } else {
        k2t_count_kernel<ChainS1><<<p.lanes, T2_THREADS, 0, c->ts>>>(p);
        t2scan_a_kernel<ChainS1><<<tiles, SCAN_BLOCK, 0, c->ts>>>(p);
        t2scan_b_kernel<ChainS1><<<1, 32, 0, c->ts>>>(p);
        t2scan_c_kernel<ChainS1><<<tiles, SCAN_BLOCK, 0, c->ts>>>(p);
        k2t_write_kernel<ChainS1><<<p.lanes, T2_THREADS, 0, c->ts>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 5;
    return WMB_OK;
}

static int launch_k2c(wmb_ctx *c, const K2cParams &p, cudaStream_t st)
{
    launch_cscan(c, p.cnt, p.base, p.lanes, p.agg, &p.sd->total, p.run_if, nullptr, 0, st, p.run_if ? 1u : 0u);
    k2c_compact_kernel<<<p.lanes, 128, 0, st>>>(p);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 1;
    return WMB_OK;
}

/* the whole gather + device framer (+ the erasure repair K4R when r is given); grids are fixed (the kernels loop over
 * however many candidates there are).  K4R adds its datagrams to pool_n, which k3_publish reads: it goes before that */
static int launch_k3_k4(wmb_ctx *c, const K3Params &p, const K4Params *q, const K4RParams *r, const K4SParams *sp)
{
    static int sms = 0;
    if (!sms) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    k3_plan_kernel<<<1, 32, 0, c->cs>>>(p);
    k3_fill_kernel<<<sms * 2, 256, 0, c->cs>>>(p);
    k3_size_kernel<<<sms, 128, 0, c->cs>>>(p);
    k3_cut_kernel<<<sms * 32, 64, 0, c->cs>>>(p);
    if (p.soft_words) {
        k3_soft_kernel<<<sms * 32, 64, 0, c->cs>>>(p);
        c->st.kernel_launches += 1;
    }
    if (p.soft_ring[WMB_CHAIN_S1 * WMB_N_ALGOS + WMB_ALGO_RLA] || p.soft_ring[WMB_CHAIN_S1 * WMB_N_ALGOS + WMB_ALGO_T2A]) {
        k3_soft_s1_kernel<<<sms * 32, 64, 0, c->cs>>>(p);     /* the S1 streams' values */
        c->st.kernel_launches += 1;
    }
    k3_offsets_kernel<<<1, SCAN_THREADS, 0, c->cs>>>(p);
    k3_copy_kernel<<<sms * 32, 128, 0, c->cs>>>(p);
    k3_carry_kernel<<<sms, 128, 0, c->cs>>>(p);
    c->st.kernel_launches += 8;
    if (q) {
        k4_decode_kernel<<<sms * 64, K4_THREADS, 0, c->cs>>>(*q);
        c->st.kernel_launches += 1;
    }
    if (r) {
        k4r_repair_kernel<<<sms * 64, K4_THREADS, 0, c->cs>>>(*r);
        c->st.kernel_launches += 1;
    }
    if (sp && (sp->k_max || sp->s_max)) {    /* C1 / T1 soft repair: overwrites K4R's record of such a candidate */
        k4s_repair_kernel<<<sms * 64, K4_THREADS, 0, c->cs>>>(*sp);
        c->st.kernel_launches += 1;
    }
    if (sp && sp->s1_max) {                  /* S1 soft repair: K4S's S1 instance */
        k4s_s1_repair_kernel<<<sms * 64, K4_THREADS, 0, c->cs>>>(*sp);
        c->st.kernel_launches += 1;
    }
    k3_publish_kernel<<<1, 32, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
    return WMB_OK;
}

static int launch_k4(wmb_ctx *c, const K4Params &p)
{
    k4_decode_kernel<<<p.n ? p.n : 1, K4_THREADS, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 1;
    return WMB_OK;
}
#endif

/* the burst pass of one chain (wmb_bursts.cuh), on cs; p.M == 0: the end-of-input gather (only kb_runs + kb_reduce) */
static int launch_bursts(wmb_ctx *c, const BurstParams &p, uint64_t *agg)
{
#ifdef WMB_HOSTSIM
    if (p.M > 0) {
        hs_for(WMB_BURST_LOOK + p.nw, [&](uint32_t wi) { kb_mask(p, wi); });
        hs_for(p.units, [&](uint32_t u) { p.cnt[u] = kb_events(p, u, false); });
        launch_cscan(c, p.cnt, p.base, p.units, agg, &p.bd->n_ev, nullptr, nullptr, 1);
        hs_for(p.units, [&](uint32_t u) { kb_events(p, u, true); });
        c->st.kernel_launches += 3;
    }
    {
        BurstRunCtx r;
        kb_run_ctx(p, r);
        static uint32_t cnt[WMB_BURST_BLOCK];
        uint32_t total = 0;
        const uint32_t chunks = (r.n_runs + WMB_BURST_BLOCK - 1) / WMB_BURST_BLOCK;
        for (uint32_t ch = 0; ch < chunks; ch++) {
            hs_for(WMB_BURST_BLOCK, [&](uint32_t t) { kb_runs_count(p, r, ch, t, cnt); });
            kb_runs_scan(cnt, &total);
            hs_for(WMB_BURST_BLOCK, [&](uint32_t t) { kb_runs_write(p, r, ch, t, cnt); });
        }
        kb_runs_finish(p, r, total);
    }
    {
        static BurstPart part[WMB_BURST_BLOCK];
        static QualAcc qpart[WMB_BURST_BLOCK];
        hs_for(p.bd->n_items, [&](uint32_t it) {
            BurstQPlan qp;
            hs_for(WMB_BURST_BLOCK, [&](uint32_t t) { kb_reduce_part(p, it, t, WMB_BURST_BLOCK, part); });
            kb_reduce_finish(p, it, part, WMB_BURST_BLOCK, p.qout ? &qp : nullptr);
            if (p.qout) {
                hs_for(WMB_BURST_BLOCK, [&](uint32_t t) { kb_qual_part(p, qp, t, WMB_BURST_BLOCK, qpart); });
                kb_qual_finish(p, it, qp, qpart, WMB_BURST_BLOCK);
            }
        });
    }
    c->st.kernel_launches += 2;
#else
    static int sms = 0;
    if (!sms) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    if (p.M > 0) {
        kb_mask_kernel<<<(WMB_BURST_LOOK + p.nw + 255) / 256, 256, 0, c->cs>>>(p);
        kb_count_kernel<<<(p.units + 255) / 256, 256, 0, c->cs>>>(p);
        launch_cscan(c, p.cnt, p.base, p.units, agg, &p.bd->n_ev, nullptr, nullptr, 1);
        kb_write_kernel<<<(p.units + 255) / 256, 256, 0, c->cs>>>(p);
        c->st.kernel_launches += 3;
    }
    kb_runs_kernel<<<1, WMB_BURST_BLOCK, 0, c->cs>>>(p);
    kb_reduce_kernel<<<sms * 4, WMB_BURST_BLOCK, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
    c->st.kernel_launches += 2;
#endif
    return WMB_OK;
}

/* the snippet pass of one batch (wmb_snippets.cuh), on cs behind the burst pass: keep flags, their ranks, the copy */
static int launch_snippets(wmb_ctx *c, const SnipParams &p, uint64_t *n_keep)
{
    const uint32_t blocks = (p.ng + WMB_SNIP_BLOCK - 1) / WMB_SNIP_BLOCK;
#ifdef WMB_HOSTSIM
    static uint8_t any[WMB_SNIP_BLOCK + WMB_SNIP_HALO];
    hs_for(blocks, [&](uint32_t b) {
        hs_for(WMB_SNIP_BLOCK + WMB_SNIP_HALO, [&](uint32_t i) { ksn_keep_fill(p, b * WMB_SNIP_BLOCK, i, any); });
        hs_for(WMB_SNIP_BLOCK, [&](uint32_t t) { ksn_keep_decide(p, b * WMB_SNIP_BLOCK, t, any); });
    });
    launch_cscan(c, p.keep, c->d_snrank, p.ng, c->d_snagg, n_keep, nullptr, nullptr, 1);
    p.sd->la1 = p.sd->la1_next;
    hs_for(p.ng, [&](uint32_t g) { hs_for(WMB_SNIP_BLOCK, [&](uint32_t t) { ksn_copy_part(p, g, t, WMB_SNIP_BLOCK); }); });
#else
    ksn_keep_kernel<<<blocks, WMB_SNIP_BLOCK, 0, c->cs>>>(p);
    launch_cscan(c, p.keep, c->d_snrank, p.ng, c->d_snagg, n_keep, nullptr, nullptr, 1);
    ksn_copy_kernel<<<p.ng, WMB_SNIP_BLOCK, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
#endif
    c->st.kernel_launches += 2;
    return WMB_OK;
}

/* the band survey's FFT pass over one batch (wmb_spectrum.cuh), on the demod stream */
static int launch_spectrum(wmb_ctx *c, const SpecParams &p, cudaStream_t st)
{
#ifdef WMB_HOSTSIM
    static SpecSmem sm;
    static SpecAcc acc[WMB_SPEC_THREADS];
    hs_for(p.n_units, [&](uint32_t gi) {
        const SpecUnit u = spec_unit(p, p.g_lo + gi);
        hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_tables(p, sm, t); ks_acc_clear(acc[t]); });
        const uint32_t L = p.logN;
        const int64_t per = WMB_SPEC_POINTS / p.N, passes = (u.bb - u.ba + per - 1) / per;
        for (int64_t pass = 0; pass < passes; pass++) {
            hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_load(p, sm, u, pass, t, L); });
            uint32_t lh = 0;
            for (; lh + 2 <= L; lh += 2) hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_stage2(sm, lh, L, t); });
            if (L & 1u) hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_stage1(sm, L - 1, L, t); });
            const uint32_t nvalid = ks_pass_blocks(u, pass, L);
            hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_power(sm, nvalid, t, acc[t], L); });
        }
        for (int pk = 0; pk < 2; pk++) {
            hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_red_put(sm, acc[t], t, pk == 1); });
            hs_for(WMB_SPEC_THREADS, [&](uint32_t t) { ks_red_flush(p, sm, u, t, pk == 1, L); });
        }
    });
    (void)st;
#else
    static int sms = 0;
    if (!sms) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    const uint32_t grid = std::min<uint32_t>(p.n_units, (uint32_t)sms * 4u);
    switch (p.logN) {                                  /* one instance per N: shifts and masks of constants */
    case 8:  ks_fft_kernel<8><<<grid, WMB_SPEC_THREADS, 0, st>>>(p); break;
    case 9:  ks_fft_kernel<9><<<grid, WMB_SPEC_THREADS, 0, st>>>(p); break;
    case 10: ks_fft_kernel<10><<<grid, WMB_SPEC_THREADS, 0, st>>>(p); break;
    default: ks_fft_kernel<11><<<grid, WMB_SPEC_THREADS, 0, st>>>(p); break;
    }
    CUDA_TRY(cudaGetLastError());
#endif
    c->st.kernel_launches++;
    return WMB_OK;
}

static int launch_spec_close(wmb_ctx *c, const SpecCloseParams &p, cudaStream_t st)
{
#ifdef WMB_HOSTSIM
    hs_for(p.n, [&](uint32_t j) { hs_for(p.N, [&](uint32_t k) { ks_close(p, j, k); }); });
    (void)st;
#else
    ks_close_kernel<<<p.n, 256, 0, st>>>(p);
    CUDA_TRY(cudaGetLastError());
#endif
    c->st.kernel_launches++;
    return WMB_OK;
}

/* --------------------------------------------------------------------------- */
/* set-up                                                                      */
/* --------------------------------------------------------------------------- */

extern "C" void wmb_default_opts(wmb_opts *o)
{
    memset(o, 0, sizeof(*o));
    o->decimation = 2;          /* rtl_wmbus.c:857 */
    o->accurate_atan = 1;       /* :859 */
    o->rla_enabled = 1;         /* :855 */
    o->t2_enabled = 1;          /* :856 */
    o->t1c1_enabled = 1;        /* :862 */
    o->s1_enabled = 1;          /* :863 */
}

extern "C" int wmb_abi_version(void) { return WMB_ABI_VERSION; }
extern "C" const char *wmb_last_error(void) { return g_err; }
extern "C" const char *wmb_version_string(void) { return WMB_VERSION; }

extern "C" void *wmb_host_alloc(size_t nbytes)
{
    void *p = nullptr;
    if (cudaMallocHost(&p, nbytes ? nbytes : 1) != cudaSuccess) {
        set_err(WMB_E_NOMEM, "cannot allocate %zu bytes of pinned host memory", nbytes);
        return nullptr;
    }
    return p;
}

extern "C" void wmb_host_free(void *p) { if (p) cudaFreeHost(p); }

static uint64_t next_pow2(uint64_t v)
{
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

template <typename T>
static int dev_alloc(wmb_ctx *c, T **p, size_t count, bool zero = false)
{
    void *q = nullptr;
    const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
    if (cudaMalloc(&q, bytes) != cudaSuccess) return set_err(WMB_E_NOMEM, "cudaMalloc of %zu bytes failed", bytes);
    if (zero && cudaMemset(q, 0, bytes) != cudaSuccess) return set_err(WMB_E_CUDA, "cudaMemset failed");
    c->dev_allocs.push_back(q);
    *p = (T *)q;
    return WMB_OK;
}

template <typename T>
static int host_alloc(wmb_ctx *c, T **p, size_t count)
{
    void *q = nullptr;
    if (cudaMallocHost(&q, std::max<size_t>(count * sizeof(T), 16)) != cudaSuccess)
        return set_err(WMB_E_NOMEM, "cudaMallocHost failed");
    c->host_allocs.push_back(q);
    *p = (T *)q;
    return WMB_OK;
}

#define TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

static int mem_free(wmb_ctx *c, void *p, bool host)
{
    if (!p) return WMB_OK;
    std::vector<void *> &v = host ? c->host_allocs : c->dev_allocs;
    v.erase(std::remove(v.begin(), v.end(), p), v.end());
    CUDA_TRY(host ? cudaFreeHost(p) : cudaFree(p));
    return WMB_OK;
}

/* d and h are set only when both arrays exist */
template <typename T>
int SlotTable<T>::alloc(wmb_ctx *c, uint32_t n_parts, size_t n_cap, uint32_t first_prefix, uint32_t grow_slack)
{
    T *dd = nullptr, *hh = nullptr;
    TRY(dev_alloc(c, &dd, (size_t)WMB_NSLOT * n_parts * n_cap));
    TRY(host_alloc(c, &hh, (size_t)WMB_NSLOT * n_parts * n_cap));
    d = dd; h = hh; parts = n_parts; cap = n_cap; slack = grow_slack; prefix = (uint32_t)std::min<size_t>(first_prefix, n_cap);
    return WMB_OK;
}

template <typename T> int SlotTable<T>::release(wmb_ctx *c)
{
    TRY(mem_free(c, d, false)); TRY(mem_free(c, h, true));
    d = h = nullptr; cap = 0;
    return WMB_OK;
}

/* lane geometry of the run-length kernels; WMBUS_B200_TUNE="t2words:p1chunk:p2records" overrides it for experiments */
static uint32_t g_p1_chunk = 2048u;      /* decimated samples per phase-1 run-length lane */
static uint32_t g_p2_records = 512u;     /* records per phase-2 lane (nominal) */
#define K2P1_CHUNK g_p1_chunk
#define K2P1_WARM  256u
#define K2P1_CAP   (K2P1_CHUNK / 5 + 2)
#define K2P2_RECORDS g_p2_records

static double wall_ms();
/* WMBUS_B200_TRACE=1: host wall-clock marks of one batch on stderr (debugging aid) */
static bool g_trace = false;
static std::vector<std::pair<const char *, double>> g_marks;
static inline void tr(const char *name) { if (g_trace) g_marks.emplace_back(name, wall_ms()); }
static void tr_dump()
{
    if (!g_trace || g_marks.empty()) return;
    fprintf(stderr, "[trace]");
    for (size_t i = 1; i < g_marks.size(); i++) fprintf(stderr, " %s %.3f", g_marks[i].first, g_marks[i].second - g_marks[i - 1].second);
    fprintf(stderr, " | total %.3f ms\n", g_marks.back().second - g_marks.front().second);
    g_marks.clear();
}

/* WMBUS_B200_PIPE_MIB: cut a long device push into batches of this size that follow each other through the device
 * like through a pipeline (run_batch).  Off by default: on the 1 GiB benchmark step, 4 x 256 MiB took more device
 * time than one batch -- the demod kernel is a persistent grid that owns every SM's register
 * file, so the clock-recovery lanes of the batch before (128 registers x 64 threads per block, one serial chain per
 * thread) only get on an SM when demod blocks retire, and whatever issue slots they win stretch their critical path.
 * Host pushes are batched by the H2D copies anyway and go through the same machinery. */
static size_t g_pipe_bytes = ~(size_t)0;

static void read_tuning()
{
#ifndef WMB_HOSTSIM
    if (const char *k = getenv("WMBUS_B200_K2A")) g_k2a_coop = strcmp(k, "scalar") != 0;
    if (const char *k = getenv("WMBUS_B200_K1_CTAS")) g_k1_ctas = atoi(k);
    if (const char *k = getenv("WMBUS_B200_FIXSEG")) g_fixseg = atoi(k);
#endif
    if (const char *b = getenv("WMBUS_B200_PIPE_MIB")) { const unsigned long v = strtoul(b, nullptr, 10); if (v >= 1 && v <= 4096) g_pipe_bytes = (size_t)v << 20; }
    if (const char *b = getenv("WMBUS_B200_P2BLK")) { const unsigned v = (unsigned)atoi(b); if (v == 32 || v == 64 || v == 128) g_p2_block = v; }
    /* the first field (formerly the time2 lane length) is parsed and ignored: the time2 kernels work on fixed tiles
     * (T2_TILE_WORDS), and tools/tune_sweep*.py keep the three-field format */
    const char *e = getenv("WMBUS_B200_TUNE");
    unsigned a = 0, b = 0, r = 0;
    if (!e || sscanf(e, "%u:%u:%u", &a, &b, &r) != 3) return;
    if (b >= 512 && b <= 65536 && b % 32 == 0) g_p1_chunk = b;
    if (r >= 32 && r <= K2P2W_THREADS * K2P2W_ITEMS) g_p2_records = r;
}

static bool bursts_on(const wmb_ctx *c);

static int ctx_alloc(wmb_ctx *c)
{
    if (c->snip_mode && !bursts_on(c))
        return set_err(WMB_E_STATE, "snippets follow the burst report: turn it on for a chain (wmb_set_bursts) before the first push");
    if (c->allocated) return WMB_OK;
    const uint32_t d = c->d;
    c->M_max = (int64_t)(c->max_batch_bytes / (2 * (size_t)d));
    const uint32_t C_min = c->C_fixed ? c->C_fixed : 8192;
    c->lanes_max = (uint32_t)(c->M_max / C_min + 2);
    c->t2_tiles_max = k2t_tiles(c->M_max);
    const size_t words_rl = (size_t)c->M_max / 4 + (size_t)c->lanes_max * (K2_EDGE_EMIT_CAP + 8) + 1024;
    c->cap_words_rl = (uint32_t)std::min<size_t>(words_rl, 0xFFFFFFFFu);
    c->ring_events = next_pow2((size_t)c->M_max / 4 + 65536 + WMB_MAXBITS);
    /* A run-length stream's ring: in the regime where the tracker's bit length has collapsed (an in-channel carrier) the
     * lanes emit up to their event buffers' capacity, 1.25 events per sample, and a burst of that is as long in a small
     * batch as in a large one.  Up to 2^26 events (128 MiB batches; the CLI's live hand-overs and its 64 MiB default) the
     * ring holds whatever the monolithic lanes of a batch can emit, so it cannot be overrun by them; larger batches keep
     * the size they were measured with, which is at least that */
    c->ring_events_rl = std::max<size_t>(c->ring_events, std::min<size_t>(next_pow2(words_rl + 65536 + WMB_MAXBITS), (size_t)1 << 26));
    if (c->o.reserved[1] & 2u) c->ring_events_rl = c->ring_events;      /* tests: reach the overrun path with a small capture */
    c->p1_lanes_max = (uint32_t)(c->M_max / K2P1_CHUNK + 2);
    c->rec_max = (size_t)c->M_max / 5 + 2 * (size_t)c->p1_lanes_max + 64;
    c->p2_lanes_max = (uint32_t)(c->rec_max / K2P2_RECORDS + 2);
    /* access-code matches and gathered frame bits scale with the batch: one candidate per 256 decimated samples, one
     * frame bit per 16 (dense traffic: a telegram every ~5000 samples; false matches: 2^-16 per bit) */
    c->cand_cap = (uint32_t)std::min<int64_t>(std::max<int64_t>(c->M_max >> 8, 1 << 16), 1 << 24);
    if (c->o.reserved[1] >> 8) c->cand_cap = std::max<uint32_t>(c->o.reserved[1] >> 8, 4u);   /* tests: force the overflow path */
    c->frame_words_cap = (uint32_t)std::min<int64_t>(std::max<int64_t>(c->M_max >> 4, 1 << 22), 1 << 28);

    TRY(dev_alloc(c, &c->d_in[0], c->max_batch_bytes + 4096));
    TRY(dev_alloc(c, &c->d_in[1], c->max_batch_bytes + 4096));
    TRY(dev_alloc(c, &c->d_hist, (size_t)k1_hist_bytes(d), true));
    TRY(dev_alloc(c, &c->d_tmp, std::max<size_t>((size_t)c->W * 4, (size_t)k1_hist_bytes(d))));
    TRY(dev_alloc(c, &c->d_lut, 2 * 4096));
    TRY(dev_alloc(c, &c->d_errors, 16, true));
    c->d_nfail = c->d_errors + 4;
    TRY(dev_alloc(c, &c->d_gd, 1, true));
    c->pend_cap = 1u << 16;                      /* candidates younger than one telegram at a batch end */
    TRY(dev_alloc(c, &c->d_rec, WMB_NSLOT, true));
    TRY(dev_alloc(c, &c->d_words, c->frame_words_cap));
    TRY(dev_alloc(c, &c->d_cut_n, c->cand_cap));
    TRY(dev_alloc(c, &c->d_k3_agg, SCAN_THREADS));
    TRY(host_alloc(c, &c->h_rec, WMB_NSLOT));
    TRY(host_alloc(c, &c->h_words, c->frame_words_cap));
    /* a slot holds the candidates of one batch and their datagrams (a datagram byte takes >= 8 shipped bit words); the
     * first prefix copies take 4096 candidates and 256 KiB of datagrams, and grow with what the batches produce */
    TRY(c->hdr.alloc(c, 1, c->cand_cap, 4096, 256));
    TRY(c->dec.alloc(c, 1, c->cand_cap, 4096, 256));
    TRY(c->pool.alloc(c, 1, c->frame_words_cap / 8 + 4 * c->cand_cap, 1u << 18, 4096));

    /* mixer look-up tables, built with the host libm exactly like the reference
     * (setup_lookup_tables_for_frequency_translation, rtl_wmbus.c:974-993) */
    if (c->o.simultaneous) {
        const int fs_khz = (int)(c->o.decimation * 800u);
        const size_t n_max = (size_t)fs_khz / 25;
        if (n_max == 0 || n_max > 4096) return set_err(WMB_E_INVAL, "-s needs 1 <= decimation <= 128");
        std::vector<float> lut(2 * 4096, 0.f);
        for (size_t n = 0; n < n_max; n++) {
            const double phi = (2. * M_PI * (25 * n)) / fs_khz;
            lut[n] = cosf(phi);
            lut[4096 + n] = -sinf(phi);
        }
        CUDA_TRY(cudaMemcpy(c->d_lut, lut.data(), lut.size() * sizeof(float), cudaMemcpyHostToDevice));
    }

    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!(c->chains & (1u << ch))) continue;
        ChainBuf &b = c->cb[ch];
        const size_t n = (size_t)c->W + (size_t)c->M_max + 512;    /* slack: block loads may run past M */
        for (int k = 0; k < 2; k++) {
            SetBuf &sb = b.set[k];
            TRY(dev_alloc(c, &sb.dphi, n));
            TRY(dev_alloc(c, &sb.rssi, n));
            TRY(dev_alloc(c, &sb.dbits, n / 32 + 64, true));      /* slack: lanes prefetch 16 words ahead */
            TRY(dev_alloc(c, &sb.sbits, n / 32 + 64, true));
            if (c->taps) TRY(dev_alloc(c, &sb.cbits, n / 32 + 64, true));
            TRY(dev_alloc(c, &sb.ia_start, c->lanes_max));
            TRY(dev_alloc(c, &sb.ia_end, c->lanes_max));
            TRY(dev_alloc(c, &sb.rerun_a, c->lanes_max, true));
        }
        TRY(dev_alloc(c, &b.ia_carry, 1));
        TRY(dev_alloc(c, &b.rl_start, c->lanes_max));
        TRY(dev_alloc(c, &b.rl_end, c->lanes_max));
        TRY(dev_alloc(c, &b.rl_carry, 1));
        TRY(dev_alloc(c, &b.rerun, c->lanes_max, true));
        TRY(dev_alloc(c, &b.lane_err, c->lanes_max, true));
        if (ch == 0 && c->two_phase && c->o.rla_enabled) {
            TRY(dev_alloc(c, &b.p1_rec, (size_t)c->p1_lanes_max * K2P1_CAP));
            TRY(dev_alloc(c, &b.p1_cnt, c->p1_lanes_max, true));
            TRY(dev_alloc(c, &b.p1_base, c->p1_lanes_max));
            TRY(dev_alloc(c, &b.p1_start, c->p1_lanes_max));
            TRY(dev_alloc(c, &b.p1_end, c->p1_lanes_max));
            TRY(dev_alloc(c, &b.p1_rerun, c->p1_lanes_max, true));
            TRY(dev_alloc(c, &b.rec_m, c->rec_max));
            TRY(dev_alloc(c, &b.rec_v, c->rec_max));
            TRY(dev_alloc(c, &b.rec_n, c->rec_max));
            TRY(dev_alloc(c, &b.p2_cnt, c->p2_lanes_max, true));
            TRY(dev_alloc(c, &b.p2_base, c->p2_lanes_max));
            TRY(dev_alloc(c, &b.pd, 1, true));
            TRY(dev_alloc(c, &b.p2_out, 1, true));
        }
        TRY(dev_alloc(c, &b.t2_tail, c->t2_tiles_max));
        TRY(dev_alloc(c, &b.t2_len, c->t2_tiles_max));
        TRY(dev_alloc(c, &b.t2_sr, c->t2_tiles_max));
        uint32_t scan_lanes = c->lanes_max > c->t2_tiles_max ? c->lanes_max : c->t2_tiles_max;
        if (c->p1_lanes_max > scan_lanes) scan_lanes = c->p1_lanes_max;
        if (c->p2_lanes_max > scan_lanes) scan_lanes = c->p2_lanes_max;
        const size_t n_agg = scan_tiles(scan_lanes) + 1;
        TRY(dev_alloc(c, &b.t2_agg_tail, n_agg));
        TRY(dev_alloc(c, &b.t2_agg_len, n_agg));
        IirState ia;
        iir_state_init(ia);
        CUDA_TRY(cudaMemcpy(b.ia_carry, &ia, sizeof(ia), cudaMemcpyHostToDevice));
        RlState rl;
        rl_state_init(rl, ch);
        CUDA_TRY(cudaMemcpy(b.rl_carry, &rl, sizeof(rl), cudaMemcpyHostToDevice));
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            Stream &s = b.s[a];
            const uint32_t nl = a == WMB_ALGO_T2A ? c->t2_tiles_max : c->lanes_max;
            if (a == WMB_ALGO_RLA) TRY(dev_alloc(c, &s.ev, c->cap_words_rl));
            TRY(dev_alloc(c, &s.cnt, nl, true));
            TRY(dev_alloc(c, &s.base, nl));
            s.ring_cap = a == WMB_ALGO_RLA ? c->ring_events_rl : c->ring_events;
            TRY(dev_alloc(c, &s.ring, s.ring_cap));
            TRY(dev_alloc(c, &s.sd, 1, true));
            TRY(dev_alloc(c, &s.cand, c->cand_cap));
            TRY(dev_alloc(c, &s.pend, c->pend_cap));
            TRY(dev_alloc(c, &s.pend_ofs, c->pend_cap));
            TRY(dev_alloc(c, &s.agg, n_agg));
        }
    }
    /* the set-up copies above are plain cudaMemcpy calls from pageable memory: make sure they have landed before any
     * kernel on the context's non-blocking streams can read them */
    CUDA_TRY(cudaDeviceSynchronize());
    c->allocated = true;
    return WMB_OK;
}

static bool bursts_on(const wmb_ctx *c)
{
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) if (c->burst_level[ch] && (c->chains & (1u << ch))) return true;
    return false;
}

/* the burst pass's buffers, at the first batch that needs them.  The record table of a slot holds every piece one
 * batch can close: pieces are disjoint and >= 256 samples long, and all but the first lie in [-G, M) */
static int burst_alloc(wmb_ctx *c)
{
    if (c->burst_allocated) return WMB_OK;
    const size_t M = (size_t)c->M_max;
    const size_t nw = M / 32 + 2, units = M / WMB_BURST_UNIT + 2;
    const size_t cap = M / 256 + 4;             /* records per slot and chain: pieces >= 256 samples of one batch */
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!(c->chains & (1u << ch))) continue;
        wmb_ctx::BurstBuf &b = c->bb[ch];
        /* events: a start needs G below samples before it, an end G after it */
        const size_t ev_cap = 2 * (M / (size_t)(burst_G((uint32_t)ch) + 1) + 2) + 64;
        TRY(dev_alloc(c, &b.mask, WMB_BURST_LOOK + nw));
        TRY(dev_alloc(c, &b.cnt, units));
        TRY(dev_alloc(c, &b.base, units));
        TRY(dev_alloc(c, &b.agg, scan_tiles((uint32_t)units) + 1));
        TRY(dev_alloc(c, &b.ev, ev_cap));
        TRY(dev_alloc(c, &b.bd, 1, true));
        TRY(dev_alloc(c, &b.items, cap + 1));
    }
    TRY(c->brec.alloc(c, WMB_N_CHAINS, cap, 64, 64));
    TRY(dev_alloc(c, &c->d_bslot, WMB_NSLOT, true));
    TRY(host_alloc(c, &c->h_bslot, WMB_NSLOT));
    CUDA_TRY(cudaDeviceSynchronize());
    c->burst_allocated = true;
    return WMB_OK;
}

/* the snippet pass's buffers, at the first gather that needs them.  A slot's pool holds at most 64 MiB (or one batch):
 * sized to the batch, a jammer that keeps every granule would pin four batches of host memory */
static int snip_alloc(wmb_ctx *c)
{
    if (c->d_snd) return WMB_OK;
    const size_t gb = (size_t)4096 * c->d;
    const size_t ng = (size_t)c->M_max / WMB_SNIP_GRAN + 2;
    c->snip_pool_gran = (uint32_t)std::max<size_t>(std::min<size_t>(WMB_SNIP_POOL_MAX, c->max_batch_bytes) / gb, 1);
    if (c->o.reserved[1] & 4u) c->snip_pool_gran = 1;      /* tests: reach the lost path with a small capture */
    TRY(dev_alloc(c, &c->d_snkeep, ng));
    TRY(dev_alloc(c, &c->d_snrank, ng));
    TRY(dev_alloc(c, &c->d_snagg, scan_tiles((uint32_t)ng) + 1));
    TRY(dev_alloc(c, &c->d_snn, WMB_NSLOT, true));
    TRY(host_alloc(c, &c->h_snn, WMB_NSLOT));
    TRY(c->snlist.alloc(c, 1, ng, 256, 64));
    TRY(c->snpool.alloc(c, 1, (size_t)c->snip_pool_gran * gb, (uint32_t)std::min<size_t>(16 * gb, (size_t)c->snip_pool_gran * gb), 0));
    for (int i = 0; i < 2; i++) CUDA_TRY(cudaEventCreateWithFlags(&c->ev_snip[i], cudaEventDisableTiming));
    TRY(dev_alloc(c, &c->d_snd, 1, true));
    CUDA_TRY(cudaDeviceSynchronize());
    return WMB_OK;
}

/* the quality report's buffers, at the first gather that needs them: beside the candidate log and the carried
 * candidates, and (when the burst report is on, so its tables exist) beside the burst records.  The sums are copied
 * side by side with the headers / records, with the prefix those have grown to */
static int qual_alloc(wmb_ctx *c)
{
    if (!c->qual.d) {
        for (int ch = 0; ch < WMB_N_CHAINS; ch++)
            for (int a = 0; a < WMB_N_ALGOS; a++)
                if (c->cb[ch].s[a].pend) TRY(dev_alloc(c, &c->cb[ch].s[a].pend_qual, c->pend_cap));
        TRY(c->qual.alloc(c, 1, c->hdr.cap, c->hdr.prefix, 256));
    }
    if (c->burst_allocated && !c->bqual.d) TRY(c->bqual.alloc(c, WMB_N_CHAINS, c->brec.cap, c->brec.prefix, 64));
    return WMB_OK;
}

/* soft values: a ring beside each T1/C1 stream's ring (and, with S1 values on, each S1 stream's), the frame words' twin,
 * and its host mirror for manual mode */
static int soft_alloc(wmb_ctx *c, bool s1)
{
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (ch == WMB_CHAIN_S1 && !s1) continue;
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            Stream &s = c->cb[ch].s[a];
            if (s.ring && !s.soft_ring) TRY(dev_alloc(c, &s.soft_ring, s.ring_cap));
        }
    }
    if (c->d_soft_words) return WMB_OK;
    TRY(dev_alloc(c, &c->d_soft_words, c->frame_words_cap));
    if (c->manual) TRY(host_alloc(c, &c->h_soft_words, c->frame_words_cap));
    return WMB_OK;
}

/* the survey's window and twiddles for N bins, in double, rounded once: hann[N] | tw[N / 2][2] */
static void spec_tables(uint32_t N, float *hann, float *tw)
{
    const double pi = 3.14159265358979323846;
    for (uint32_t n = 0; n < N; n++) hann[n] = (float)(0.5 - 0.5 * cos(2.0 * pi * (double)n / (double)N));
    for (uint32_t k = 0; k < N / 2; k++) {
        tw[2 * k] = (float)cos(2.0 * pi * (double)k / (double)N);
        tw[2 * k + 1] = (float)-sin(2.0 * pi * (double)k / (double)N);
    }
}

/* rows of the ring and of a slot table: a batch closes the record left open before it and all but the last of its
 * own, and touches at most batch blocks / B + 2 consecutive records */
static uint32_t spec_rows_for(const wmb_ctx *c, uint32_t N, uint32_t B)
{
    return (uint32_t)(c->max_batch_bytes / (2 * (size_t)N) / B + 2);
}

/* the survey's buffers, at the first batch that needs them (again when a new setting needs larger tables) */
static int spec_alloc(wmb_ctx *c)
{
    const uint32_t N = c->spec_bins;
    c->spec_R = spec_rows_for(c, N, c->spec_B);
    const size_t need = (size_t)c->spec_R * N;
    if (need > c->speak.cap) {                       /* speak comes last: its cap is that of the rings and of ssum */
        CUDA_TRY(cudaDeviceSynchronize());
        TRY(mem_free(c, c->d_ssum_ring, false)); TRY(mem_free(c, c->d_speak_ring, false));
        TRY(c->ssum.release(c)); TRY(c->speak.release(c));
        TRY(dev_alloc(c, &c->d_ssum_ring, need, true));
        TRY(dev_alloc(c, &c->d_speak_ring, need, true));
        TRY(c->ssum.alloc(c, 1, need, 0, 0));         /* copied exactly: the host knows the rows a batch closed */
        TRY(c->speak.alloc(c, 1, need, 0, 0));
    }
    if (!c->d_spec_tab) {
        TRY(dev_alloc(c, &c->d_spec_tab, 2 * (size_t)WMB_SPEC_MAXN));
        cudaEventCreateWithFlags(&c->ev_spec, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&c->ev_spec_flush, cudaEventDisableTiming);
    }
    if (c->spec_tab_n != N) {
        std::vector<float> tab(2 * (size_t)N);
        spec_tables(N, tab.data(), tab.data() + N);
        CUDA_TRY(cudaMemcpy(c->d_spec_tab, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
        c->spec_tab_n = N;
    }
    return WMB_OK;
}

extern "C" int wmb_create(const wmb_opts *o, int cuda_device, wmb_ctx **out)
{
    if (!o || !out) return set_err(WMB_E_INVAL, "null argument");
    *out = nullptr;
    read_tuning();
    g_trace = getenv("WMBUS_B200_TRACE") != nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return set_err(WMB_E_NODEVICE, "no CUDA device available (libwmbus_b200 has no CPU fallback)");
    if (cuda_device < 0 || cuda_device >= ndev) return set_err(WMB_E_NODEVICE, "CUDA device %d of %d", cuda_device, ndev);
    /* the demod block stages one tile of raw samples (twice) and its converted words in shared memory: 8 bytes per input
     * sample of a 1024-row tile.  227 KB per block hold that up to decimation 25 (20 MS/s input; an RTL-SDR delivers 3.2) */
    if (o->decimation > WMB_MAX_DECIMATION)
        return set_err(WMB_E_INVAL, "decimation %u not supported (max %u: 20 MS/s input)", o->decimation, (unsigned)WMB_MAX_DECIMATION);
    if (o->simultaneous && o->decimation == 0) return set_err(WMB_E_INVAL, "-s with -d 0 is undefined in the reference");
    if (o->simultaneous > 2) return set_err(WMB_E_INVAL, "simultaneous: 0, 1 (-s) or 2 (explicit carriers)");
    if (o->prefilter > 4) return set_err(WMB_E_INVAL, "prefilter: 0 (moving averages), 1 (23-tap FIR), 2 (polyphase), 3 / 4 (their fixed-point twins)");
    if (o->prefilter && o->decimation != 2) return set_err(WMB_E_INVAL, "the pre-decimation low-passes are 1.6 MS/s designs: decimation must be 2");
    if (o->simultaneous == 2)
        for (int ch = 0; ch < 2; ch++)
            if (o->carrier_25khz[ch] == INT32_MIN || 2 * (o->carrier_25khz[ch] < 0 ? -o->carrier_25khz[ch] : o->carrier_25khz[ch]) > (int32_t)(o->decimation * 32u))
                return set_err(WMB_E_INVAL, "carrier offset outside the sampled band (|offset| <= fs / 2)");
    CUDA_TRY(cudaSetDevice(cuda_device));

    wmb_ctx *c = new wmb_ctx();
    c->o = *o;
    c->device = cuda_device;
    c->d = o->decimation ? o->decimation : 1;               /* rtl_wmbus.c:1350-1352: d==0 keeps every sample */
    c->chains = (o->t1c1_enabled ? 1u : 0u) | (o->s1_enabled ? 2u : 0u);
    /* warm-up (decimated samples) of the speculative lanes: the clock biquads need ~20 k
     * samples to re-join the true trajectory bit for bit (SURVEY.md A.7), the DC block
     * another ~18 k in front of them (A.6); a run-length lane must reach back past the
     * start of the telegram it may begin in (A.8: <= 28 k samples T1, <= 113 k S1). */
    if (o->warmup_samples) {
        c->W_a[0] = c->W_a[1] = c->W_m[0] = c->W_m[1] = (o->warmup_samples + 255) / 256 * 256;
    } else {
        /* measured re-join times of the biquad state (tools/ + DESIGN.md): T1/C1 filter <= 19 k samples,
         * S1 filter (22-42 kHz band) <= 55 k; the DC block adds its own ~18 k in front */
        c->W_a[0] = o->remove_dc ? 98304u : 24576u;    /* measured re-join <= 19k samples; a miss only costs a re-run */
        c->W_a[1] = o->remove_dc ? 163840u : 81920u;   /* 0 / 32 / 96 re-runs of 0.3 M lanes at 81920 / 65536 / 57344 */
        /* run-length lanes.  T1/C1: the PI bit-length tracker remembers the whole reset-free stretch, so a cold
         * start re-joins at the first reset both trajectories share, at the latest when the telegram it started
         * in is over (<= 28 k samples).  S1: the state is the average run length of the last low and the last
         * high run plus 24 emitted bits, so it re-joins within ~30 runs; measured on the GPU: 0 / 0 / 64 / 248
         * re-runs of 0.3 M lanes at 16384 / 4096 / 2048 / 1024 samples. */
        c->W_m[0] = 32768u; c->W_m[1] = 8192u;
    }
    c->W = 0;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!(c->chains & (1u << ch))) continue;
        c->W = std::max(c->W, c->W_a[ch]);
        if (o->rla_enabled) c->W = std::max(c->W, c->W_m[ch]);
    }
    /* the carrier-offset window of a match early in a batch reaches back into the dphi history prefix (S1: 1367
     * samples).  A longer prefix changes no lane: they reach back W_a / W_m samples, clipped at the first sample pushed */
    static_assert(WMB_OFS_HIST >= WMB_OFS_S1_LO && WMB_OFS_HIST >= WMB_OFS_T1C1_LO && WMB_OFS_HIST % 256 == 0,
                  "the dphi history prefix must hold the longest carrier-offset window, in whole lane words");
    c->W = std::max<uint32_t>(c->W, WMB_OFS_HIST);
    {
        /* DC gain of the post-demod FIR, from the tables the demod kernel uses */
        float t[2][46];
#ifdef WMB_HOSTSIM
        memcpy(t[0], c_fir_t1c1, sizeof(c_fir_t1c1));
        memcpy(t[1], c_fir_s1, sizeof(c_fir_s1));
#else
        if (cudaMemcpyFromSymbol(t[0], c_fir_t1c1, sizeof(c_fir_t1c1)) != cudaSuccess ||
            cudaMemcpyFromSymbol(t[1], c_fir_s1, sizeof(c_fir_s1)) != cudaSuccess) {
            delete c;
            return set_err(WMB_E_CUDA, "cannot read the FIR tables");
        }
#endif
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            const int nt = ch == 0 ? ChainT1C1::NTAPS : ChainS1::NTAPS;
            double g = 0.0;
            for (int i = 0; i < nt; i++) g += (double)t[ch][i];
            c->fir_gain[ch] = g;
        }
    }
    c->manual = o->manual_frames != 0;
    c->taps = (o->reserved[1] & 1u) != 0;
    c->two_phase = o->reserved[0] == 0;                  /* reserved[0] = 1: force the monolithic run-length lanes (tests) */
    c->C_fixed = o->chunk_samples ? (o->chunk_samples + 255) / 256 * 256 : 0;
    if (c->C_fixed && (c->C_fixed < 1024 || c->C_fixed > K2_MAX_CHUNK)) { delete c; return set_err(WMB_E_INVAL, "chunk_samples out of range"); }
    size_t mb = o->max_batch_mib ? (size_t)o->max_batch_mib * 1048576u : (size_t)256 * 1048576u;
    const size_t gran = (size_t)4096 * c->d;
    mb = (mb + gran - 1) / gran * gran;
    c->max_batch_bytes = mb;
    memset(&c->st, 0, sizeof(c->st));
    if (cudaStreamCreateWithFlags(&c->cs, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->xs, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->k1s, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->as[0], cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->as[1], cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->as2[0], cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->as2[1], cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->ts, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->s2, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->rs, cudaStreamNonBlocking) != cudaSuccess) {
        delete c;
        return set_err(WMB_E_CUDA, "cannot create CUDA streams");
    }
    for (int i = 0; i < 2; i++) {
        cudaEventCreate(&c->ev_h2d[i]); cudaEventCreate(&c->ev_k1done[i]);
        cudaEventCreateWithFlags(&c->ev_k1[i], cudaEventDisableTiming); cudaEventCreateWithFlags(&c->ev_k2a[i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&c->ev_chain[i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&c->ev_k2a2[i], cudaEventDisableTiming);
    }
    cudaEventCreate(&c->ev_push_start);
    cudaEventCreateWithFlags(&c->ev_reset, cudaEventDisableTiming);
    for (int i = 0; i < WMB_NSLOT; i++) {
        cudaEventCreateWithFlags(&c->ev_res[i], cudaEventDisableTiming);
        for (int k = 0; k < 6; k++) cudaEventCreate(&c->ev_t[i][k]);
    }
    cudaEventCreate(&c->ev_fork);
    cudaEventCreate(&c->ev_join);
    cudaEventCreate(&c->ev_fork2);
    cudaEventCreate(&c->ev_join2);
    cudaEventCreateWithFlags(&c->ev_join_rs, cudaEventDisableTiming);
    *out = c;
    return WMB_OK;
}

extern "C" void wmb_destroy(wmb_ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->cs) cudaStreamSynchronize(c->cs);
    if (c->xs) cudaStreamSynchronize(c->xs);
    for (void *p : c->dev_allocs) cudaFree(p);
    for (void *p : c->host_allocs) cudaFreeHost(p);
    for (cudaStream_t st : { c->k1s, c->as[0], c->as[1], c->as2[0], c->as2[1], c->ts, c->s2, c->rs }) if (st) cudaStreamSynchronize(st);
    for (int i = 0; i < 2; i++) {
        for (cudaEvent_t e : { c->ev_h2d[i], c->ev_k1done[i], c->ev_k1[i], c->ev_k2a[i], c->ev_k2a2[i], c->ev_chain[i], c->ev_snip[i] }) if (e) cudaEventDestroy(e);
        if (c->as[i]) cudaStreamDestroy(c->as[i]);
        if (c->as2[i]) cudaStreamDestroy(c->as2[i]);
    }
    if (c->k1s) cudaStreamDestroy(c->k1s);
    if (c->ev_push_start) cudaEventDestroy(c->ev_push_start);
    if (c->ev_reset) cudaEventDestroy(c->ev_reset);
    if (c->ev_spec) cudaEventDestroy(c->ev_spec);
    if (c->ev_spec_flush) cudaEventDestroy(c->ev_spec_flush);
    for (int i = 0; i < WMB_NSLOT; i++) {
        if (c->ev_res[i]) cudaEventDestroy(c->ev_res[i]);
        for (int k = 0; k < 6; k++) if (c->ev_t[i][k]) cudaEventDestroy(c->ev_t[i][k]);
    }
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    if (c->ts) cudaStreamDestroy(c->ts);
    if (c->ev_fork2) cudaEventDestroy(c->ev_fork2);
    if (c->ev_join2) cudaEventDestroy(c->ev_join2);
    if (c->s2) cudaStreamDestroy(c->s2);
    if (c->ev_join_rs) cudaEventDestroy(c->ev_join_rs);
    if (c->rs) cudaStreamDestroy(c->rs);
    if (c->cs) cudaStreamDestroy(c->cs);
    if (c->xs) cudaStreamDestroy(c->xs);
    delete c;
}

/* --------------------------------------------------------------------------- */
/* one batch on the device                                                     */
/* --------------------------------------------------------------------------- */

/* The history prefix of a [W | batch] array of the set the next batch will use <- the last W elements the previous
 * batch left in its set (element size es, prev_M elements in the previous batch).  Source and destination are different
 * allocations, so one copy does. */
static int copy_history(void *dst, const void *src_set, size_t es, int64_t W, int64_t prev_M, cudaStream_t st)
{
    if (W <= 0) return WMB_OK;
    CUDA_TRY(cudaMemcpyAsync(dst, (const uint8_t *)src_set + (size_t)prev_M * es, (size_t)W * es, cudaMemcpyDeviceToDevice, st));
    return WMB_OK;
}

static uint32_t pick_chunk(const wmb_ctx *c, int64_t M, bool alone)
{
    if (c->C_fixed) return c->C_fixed;
    /* The clock-recovery lanes are bound by the fp32 pipe of the scheduler they sit on, so a batch that has the GPU to
     * itself is cut into about one warp per scheduler (H100: 132 SMs x 4 x 32 lanes).  A batch that is followed by
     * another one overlaps its lanes with that batch's demod kernel: their latency is hidden, what counts is the
     * redundant warm-up arithmetic, so the lanes are made longer. */
    int64_t C = (M + 16895) / 16896;
    C = (C + 1023) / 1024 * 1024;
    /* A small batch on its own (a live stream's 100 ms hand-over) is all latency: its lanes take warm-up + C steps
     * however few they are, so they are made as short as the per-lane buffers allow (sized for lanes of 8192 samples at
     * the largest batch). */
    int64_t lo = alone ? 1024 : 16384;
    if (alone && c->lanes_max > 2) {
        const int64_t need = (M + c->lanes_max - 3) / (c->lanes_max - 2);
        lo = std::max<int64_t>(lo, (need + 1023) / 1024 * 1024);
    }
    if (C < lo) C = lo;
    if (C > 65536) C = 65536;
    return (uint32_t)C;
}

/* Lane length of the clock-recovery kernel when three threads share a lane (k2a2_lanes_kernel).  A lone warp takes
 * ~13 cycles per warm-up step and ~21 per live step (a second warp on the same scheduler doubles that: the kernel is
 * issue-bound with two), against 59 for the per-thread kernel -- so the batch is cut into ONE warp (ten lanes) per
 * scheduler, on H100 132 SMs x 4 x 10 lanes, and the 24576-sample warm-up is paid 5280 times instead of 16896 times. */
static uint32_t pick_chunk_coop(const wmb_ctx *c, int64_t M)
{
    if (c->C_fixed) return c->C_fixed;
    int64_t C = (M + 5279) / 5280;
    C = (C + 255) / 256 * 256;
    if (C < 8192) C = 8192;
    if (C > 131072) C = 131072;
    return (uint32_t)C;
}

/* a survey record's row: `blocks` of its blocks counted */
static wmb_spectrum_row spec_row(const wmb_ctx *c, int64_t record, uint32_t blocks)
{
    const uint64_t N = c->spec_bins, B = c->spec_B;
    const double fs = 0.8e6 * (double)c->d;
    wmb_spectrum_row w;
    memset(&w, 0, sizeof(w));
    w.record = (uint64_t)record; w.start_iq = (uint64_t)record * B * N; w.blocks = blocks; w.bins = (uint32_t)N;
    w.hz_low = -fs / 2; w.hz_step = fs / (double)N;
    return w;
}

/* Enqueue the per-sample device pass for one batch whose bytes are at `src` (device memory): demod on k1s, clock
 * recovery lanes on as[set], everything that is sequential from batch to batch on cs.  Nothing here waits for the
 * device: refuted speculative lanes are re-run by on-device fix-up kernels, and the fallback from the two-phase
 * run-length path to the monolithic lanes is a set of kernels that do nothing unless the device flag asks for them.
 * input_ready: event after which `src` holds the bytes (H2D copy), or null.  alone: no batch follows in this push. */
/* the band survey of one batch (IQ samples [q0, q0 + n_iq), bytes at src), on the demod stream sk while the batch's
 * input is still valid: the FFT pass over its counted blocks, then the rows it closes -> the slot rows, zeroed in the
 * ring.  The host knows which blocks count and which records close; the rows wait in spec_batch_rows for the gather. */
static int spec_batch(wmb_ctx *c, const uint8_t *src, uint64_t q0, uint64_t n_iq, cudaStream_t sk, int slot)
{
    const uint64_t N = c->spec_bins, B = c->spec_B;
    const int64_t p0 = (int64_t)(q0 / N), p1 = (int64_t)((q0 + n_iq) / N);
    c->spec_batch_rows.clear();
    if (p1 <= p0) return WMB_OK;
    TRY(spec_alloc(c));
    if (c->spec_flush_pending) { CUDA_TRY(cudaStreamWaitEvent(sk, c->ev_spec_flush, 0)); c->spec_flush_pending = false; }
    /* floor(b N / d) in [win_lo, win_hi)  <=>  b in [ceil(win_lo d / N), ceil(win_hi d / N)) */
    auto first_b = [&](uint64_t m) {
        const unsigned __int128 x = ((unsigned __int128)m * c->d + N - 1) / N;
        return x > (unsigned __int128)INT64_MAX ? INT64_MAX : (int64_t)x;
    };
    const int64_t c0 = std::max(p0, first_b(c->win_lo)), c1 = std::min(p1, first_b(c->win_hi));
    const int64_t r_last = (p1 - 1) / (int64_t)B;
    auto counted = [&](int64_t r) {
        const int64_t lo = std::max(c0, r * (int64_t)B), hi = std::min(c1, (r + 1) * (int64_t)B);
        return (uint32_t)(hi > lo ? hi - lo : 0) + (r == c->spec_open ? c->spec_open_blocks : 0u);
    };
    int64_t lone = -1, r_lo = 0, r_hi = 0;          /* closed: lone (if any), then records [r_lo, r_hi) */
    int64_t open = -1;
    if (c1 > c0) {
        SpecParams p;
        memset(&p, 0, sizeof(p));
        p.in = src; p.b_first = p0; p.c0 = c0; p.c1 = c1;
        p.N = (uint32_t)N; p.logN = (uint32_t)__builtin_ctz((uint32_t)N); p.B = (uint32_t)B;
        /* units: about 4 per SM-resident CTA slot of the largest batch; any size gives the same sums and maxima */
        const uint32_t per = WMB_SPEC_POINTS / (uint32_t)N;
        const uint64_t G = std::max<uint64_t>(per, ((uint64_t)(c1 - c0) / 2048 + per - 1) / per * per);
        p.G = (uint32_t)std::min<uint64_t>(G, B); p.U = (uint32_t)((B + p.G - 1) / p.G);
        p.g_lo = (c0 / (int64_t)B) * p.U + (c0 % (int64_t)B) / p.G;
        const int64_t g_hi = ((c1 - 1) / (int64_t)B) * p.U + ((c1 - 1) % (int64_t)B) / p.G;
        p.n_units = (uint32_t)(g_hi - p.g_lo + 1);
        p.R = c->spec_R; p.hann = c->d_spec_tab; p.tw = c->d_spec_tab + N;
        p.sum = c->d_ssum_ring; p.peak = c->d_speak_ring;
        TRY(launch_spectrum(c, p, sk));
        const int64_t rc0 = c0 / (int64_t)B, rc1 = (c1 - 1) / (int64_t)B;
        if (c->spec_open >= 0 && c->spec_open != rc0) lone = c->spec_open;
        r_lo = rc0; r_hi = std::min(rc1 + 1, r_last);
        if (rc1 == r_last) open = rc1;
    } else if (c->spec_open >= 0) {
        if (c->spec_open < r_last) lone = c->spec_open; else open = c->spec_open;
    }
    if (lone >= 0) c->spec_batch_rows.push_back(spec_row(c, lone, counted(lone)));
    for (int64_t r = r_lo; r < r_hi; r++) c->spec_batch_rows.push_back(spec_row(c, r, counted(r)));
    const uint32_t open_blocks = open >= 0 ? counted(open) : 0u;
    if (!c->spec_batch_rows.empty()) {
        SpecCloseParams q;
        memset(&q, 0, sizeof(q));
        q.sum = c->d_ssum_ring; q.peak = c->d_speak_ring;
        q.out_sum = c->ssum.d + c->ssum.at(slot); q.out_peak = c->speak.d + c->speak.at(slot);
        q.lone = lone; q.r_lo = r_lo; q.n = (uint32_t)c->spec_batch_rows.size(); q.N = (uint32_t)N; q.R = c->spec_R;
        TRY(launch_spec_close(c, q, sk));
    }
    c->spec_open = open; c->spec_open_blocks = open_blocks;
    CUDA_TRY(cudaEventRecord(c->ev_spec, sk));
    c->spec_enqueued = true;
    return WMB_OK;
}

static int run_batch(wmb_ctx *c, const uint8_t *src, size_t nbytes, cudaEvent_t input_ready, bool alone)
{
    tr("batch-start");
    const uint32_t d = c->d;
    const int64_t n_iq = (int64_t)(nbytes / 2);
    const int64_t M = n_iq / d;
    if (M <= 0) return WMB_OK;
    const int set = (int)(c->batch_no & 1u), pset = set ^ 1;
    const int slot = (int)(c->gather_no % WMB_NSLOT);           /* the gather that follows this batch */
    cudaEvent_t *evt = c->ev_t[slot];
    const bool first = c->batch_no == 0;
    /* a batch with nothing before it in flight and nothing behind it has nobody to overlap with: its demod kernel and
     * clock lanes go on cs too, which saves the cross-stream hand-overs (a few microseconds each) */
    const bool solo = alone && c->inflight.empty();
    cudaStream_t sk = solo ? c->cs : c->k1s, sa = solo ? c->cs : c->as[set];
    if (c->reset_pending) {                            /* the streams that do not follow cs wait for wmb_reset's kernel */
        for (cudaStream_t st : { c->k1s, c->as[0], c->as[1], c->as2[0], c->as2[1] }) CUDA_TRY(cudaStreamWaitEvent(st, c->ev_reset, 0));
        c->reset_pending = false;
    }
    const bool any_sync = c->o.rla_enabled || c->o.t2_enabled;
    /* the demod kernel slices the data bits unless the DC block (-o) sits between its FIR and the slicer */
    const bool k1_bits = any_sync && !c->o.remove_dc;
    /* ================= stage 1 (k1s): history prefix of this set, demod ================= */
    if (c->chain_recorded[set]) CUDA_TRY(cudaStreamWaitEvent(sk, c->ev_chain[set], 0));    /* batch i-2 is done with the set */
    if (input_ready) CUDA_TRY(cudaStreamWaitEvent(sk, input_ready, 0));
    if (!first)
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(c->chains & (1u << ch))) continue;
            ChainBuf &b = c->cb[ch];
            TRY(copy_history(b.set[set].dphi, b.set[pset].dphi, 4, c->W, c->prev_M, sk));
            TRY(copy_history(b.set[set].rssi, b.set[pset].rssi, 1, c->W, c->prev_M, sk));
            /* bit history for the run-length warm-ups: the previous batch's last W samples */
            if (k1_bits && c->prev_M % 32 == 0)          /* only a final (flush) batch can be ragged */
                TRY(copy_history(b.set[set].dbits, b.set[pset].dbits, 4, c->W / 32, c->prev_M / 32, sk));
        }
    CUDA_TRY(cudaEventRecord(evt[0], sk));
    if (!c->push_started) { CUDA_TRY(cudaEventRecord(c->ev_push_start, sk)); c->push_started = true; }
    K1Params k1;
    memset(&k1, 0, sizeof(k1));
    k1.in = src; k1.hist = c->d_hist; k1.in_bytes = (int64_t)nbytes;
    k1.n_hist_iq = c->hist_iq;
    k1.M = M; k1.d = d; k1.chains = c->chains;
    k1.accurate = c->o.accurate_atan; k1.mix = c->o.simultaneous ? 1u : 0u;
    k1.prefilter = c->o.prefilter;
    k1.rpt = k1_rows_per_thread(d, k1.mix, k1.prefilter);
    k1.lut_n = c->o.simultaneous ? (c->o.decimation * 800u) / 25u : 1u;
    k1.mix_k0 = (uint32_t)(c->iq_consumed % k1.lut_n);
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        /* the reference's -s: T1/C1 chain 325 kHz above the centre, S1 chain 325 kHz below (rtl_wmbus.c:1008, :1025-1030) */
        const int32_t off = c->o.simultaneous == 2 ? c->o.carrier_25khz[ch] : (ch == 0 ? 13 : -13);
        const uint32_t mag = (uint32_t)(off < 0 ? -(int64_t)off : (int64_t)off);
        k1.mix_step[ch] = mag % k1.lut_n;
        k1.mix_conj[ch] = off < 0 ? 1u : 0u;
    }
    k1.lut_cos = c->d_lut; k1.lut_msin = c->d_lut + 4096;
    k1.tile_ctr = c->d_errors + 12;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        k1.dphi[ch] = c->cb[ch].set[set].dphi ? c->cb[ch].set[set].dphi + c->W : nullptr;
        k1.rssi[ch] = c->cb[ch].set[set].rssi ? c->cb[ch].set[set].rssi + c->W : nullptr;
        k1.dbits[ch] = k1_bits && c->cb[ch].set[set].dbits ? c->cb[ch].set[set].dbits + c->W / 32 : nullptr;
    }
    TRY(launch_demod(c, k1, sk));
    CUDA_TRY(cudaEventRecord(evt[1], sk));
    CUDA_TRY(cudaEventRecord(c->ev_k1[set], sk));
    /* keep the last k1_hist_bytes() of the stream for the next batch's tile 0 */
    {
        const size_t hb = (size_t)k1_hist_bytes(d);
        if (nbytes >= hb) {
            CUDA_TRY(cudaMemcpyAsync(c->d_hist, src + nbytes - hb, hb, cudaMemcpyDeviceToDevice, sk));
        } else {
            CUDA_TRY(cudaMemcpyAsync(c->d_tmp, c->d_hist + nbytes, hb - nbytes, cudaMemcpyDeviceToDevice, sk));
            CUDA_TRY(cudaMemcpyAsync(c->d_tmp + (hb - nbytes), src, nbytes, cudaMemcpyDeviceToDevice, sk));
            CUDA_TRY(cudaMemcpyAsync(c->d_hist, c->d_tmp, hb, cudaMemcpyDeviceToDevice, sk));
        }
        c->hist_iq = std::min<int64_t>(c->hist_iq + n_iq, (int64_t)hb / 2);
    }
    /* the band survey reads the input in place */
    if (c->spec_bins) TRY(spec_batch(c, src, c->iq_consumed, (uint64_t)n_iq, sk, slot));
    /* the input buffer may be overwritten by the next H2D from here on */
    CUDA_TRY(cudaEventRecord(c->ev_k1done[c->buf_idx], sk));

    const uint32_t C = pick_chunk(c, M, alone);
    const uint32_t lanes = (uint32_t)((M + C - 1) / C);
    if (lanes > c->lanes_max) return set_err(WMB_E_INVAL, "internal: %u lanes > %u", lanes, c->lanes_max);
    const int64_t wofs = c->W / 32;                       /* word offset of batch sample 0 */

    /* ---- run-length bit sync: T1/C1 on st0, S1 on st1 ---- */
    auto enqueue_run_length = [&](cudaStream_t st0, cudaStream_t st1) -> int {
        const bool two = (c->chains & 1u) && c->two_phase;
        /* chains that take the monolithic lanes unconditionally: S1 always, T1/C1 when forced (tests) */
        const uint32_t mono = (c->chains & 2u) | (((c->chains & 1u) && !two) ? 1u : 0u);
        K2mParams km[WMB_N_CHAINS];
        auto setup_mono = [&](int ch, const uint32_t *run_if) -> int {
            ChainBuf &b = c->cb[ch];
            SetBuf &sb = b.set[set];
            K2mParams &p = km[ch];
            memset(&p, 0, sizeof(p));
            p.dbits = sb.dbits + wofs; p.rssi = sb.rssi + c->W; p.M = M; p.hist = c->hist_m;
            p.C = C; p.W = c->W_m[ch]; p.lanes = lanes;
            p.cap = C / 4 + K2_EDGE_EMIT_CAP + 8;
            if ((uint64_t)lanes * p.cap > c->cap_words_rl) return set_err(WMB_E_INVAL, "internal: event buffers too small for C=%u", C);
            p.ev = b.s[WMB_ALGO_RLA].ev; p.cnt = b.s[WMB_ALGO_RLA].cnt;
            p.st_start = b.rl_start; p.st_end = b.rl_end; p.carry = b.rl_carry; p.rerun = b.rerun;
            p.errors = c->d_errors; p.lane_err = b.lane_err;
            p.mode = 0; p.run_if = run_if; p.ac_err = c->ac_err[ch];
            if (!run_if) c->st.lanes_run += lanes;
            return WMB_OK;
        };
        auto compact_mono = [&](int ch, cudaStream_t st, const uint32_t *run_if) -> int {       /* lane events -> ring */
            ChainBuf &b = c->cb[ch];
            Stream &s = b.s[WMB_ALGO_RLA];
            K2cParams q;
            memset(&q, 0, sizeof(q));
            q.ev = s.ev; q.cnt = s.cnt; q.base = s.base; q.lanes = lanes; q.cap = km[ch].cap; q.C = C;
            q.m_base = (int64_t)c->m_consumed;
            q.ring = s.ring; q.ring_mask = s.ring_cap - 1; q.sd = s.sd; q.cand = s.cand; q.cand_cap = c->cand_cap;
            q.agg = s.agg; q.rssi = b.set[set].rssi + c->W; q.run_if = run_if;
            q.lane_err = b.lane_err; q.errors = c->d_errors;
            return launch_k2c(c, q, st);
        };
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(mono & (1u << ch))) continue;
            cudaStream_t st = ch == 0 ? st0 : st1;
            TRY(setup_mono(ch, nullptr));
            TRY(launch_k2m(c, ch, km[ch], st));
            TRY(launch_k2m_carry(c, c->cb[ch].rl_end + (lanes - 1), c->cb[ch].rl_carry, nullptr, st));
            TRY(compact_mono(ch, st, nullptr));
        }
        if (two) {
            /* T1/C1: phase 1 (per-sample, verified) -> records -> phase 2 (per-run) */
            ChainBuf &b = c->cb[0];
            Stream &s = b.s[WMB_ALGO_RLA];
            K2p1Params p1;
            memset(&p1, 0, sizeof(p1));
            p1.dbits = b.set[set].dbits + wofs; p1.M = M; p1.hist = c->hist_m;
            p1.C = K2P1_CHUNK; p1.W = K2P1_WARM; p1.lanes = (uint32_t)((M + K2P1_CHUNK - 1) / K2P1_CHUNK);
            p1.cap = K2P1_CAP; p1.rec = b.p1_rec; p1.cnt = b.p1_cnt;
            p1.st_start = b.p1_start; p1.st_end = b.p1_end; p1.carry = b.rl_carry; p1.rerun = b.p1_rerun;
            p1.mode = 0;
            if (p1.lanes > c->p1_lanes_max) return set_err(WMB_E_INVAL, "internal: phase-1 lanes");
            c->st.lanes_run += p1.lanes;
            TRY(launch_k2p1(c, p1, st0));
            K2pcParams pc;
            memset(&pc, 0, sizeof(pc));
            pc.rec = b.p1_rec; pc.cnt = b.p1_cnt; pc.base = b.p1_base; pc.lanes = p1.lanes; pc.cap = p1.cap; pc.C = p1.C;
            pc.rec_m = b.rec_m; pc.rec_v = b.rec_v; pc.agg = s.agg; pc.pd = b.pd;
            K2p2Params p2;
            memset(&p2, 0, sizeof(p2));
            p2.rec_m = b.rec_m; p2.rec_v = b.rec_v; p2.rec_n = b.rec_n; p2.pd = b.pd; p2.R = K2P2_RECORDS;
            p2.lanes = (uint32_t)(((uint64_t)M / 5 + 2 * (uint64_t)p1.lanes) / K2P2_RECORDS + 2);
            if (p2.lanes > c->p2_lanes_max) return set_err(WMB_E_INVAL, "internal: phase-2 lanes");
            p2.cnt = b.p2_cnt; p2.base = b.p2_base; p2.rssi = b.set[set].rssi + c->W; p2.m_base = (int64_t)c->m_consumed;
            p2.ring = s.ring; p2.ring_mask = s.ring_cap - 1; p2.sd = s.sd; p2.cand = s.cand; p2.cand_cap = c->cand_cap;
            p2.carry = b.rl_carry; p2.p2_out = b.p2_out; p2.agg = s.agg; p2.ac_err = c->ac_err[0];
            TRY(launch_k2p_rest(c, pc, p2, st0));
            /* the second reset rule (rtl_wmbus.c:756-762) fired somewhere in this batch (pd->fallback, set by phase
             * 2, which then wrote nothing): redo T1/C1 with the exact monolithic lanes.  The kernels are always
             * enqueued; without the flag every thread returns at once. */
            const uint32_t *flag = &b.pd->fallback;
            TRY(setup_mono(0, flag));
            TRY(launch_k2m(c, 0, km[0], st0));
            TRY(compact_mono(0, st0, flag));
            TRY(launch_k2p_fold(c, b.p1_end + (p1.lanes - 1), b.p2_out, b.rl_carry, b.pd, b.rl_end + (lanes - 1), st0));
        }
        return WMB_OK;
    };

    if (any_sync) {
        const bool coop = c->o.t2_enabled && !c->o.remove_dc && M % 32 == 0;
        /* The run-length path reads only the data bits and the rssi, both from the demod kernel here: it starts right
         * behind that kernel, T1/C1 on rs and S1 on s2, and runs beside the clock lanes (one warp per scheduler,
         * mostly idle SMs), instead of after their verification.  Both streams also wait for what cs held before this
         * batch -- the previous gather reads the rings and candidate lists these kernels append to, wmb_reset's
         * kernel sets their carries -- and cs waits for them before the gather (ev_chain[set] thus covers them too).
         * -o (the clock lanes slice), a ragged final batch and a batch without time2 keep the order below. */
        const bool early = coop && c->o.rla_enabled;
        if (early) {
            CUDA_TRY(cudaEventRecord(c->ev_fork2, c->cs));
            for (cudaStream_t st : { c->rs, c->s2 }) {
                CUDA_TRY(cudaStreamWaitEvent(st, c->ev_fork2, 0));
                CUDA_TRY(cudaStreamWaitEvent(st, c->ev_k1[set], 0));
            }
            TRY(enqueue_run_length(c->rs, c->s2));
            CUDA_TRY(cudaEventRecord(c->ev_join_rs, c->rs));
            CUDA_TRY(cudaEventRecord(c->ev_join2, c->s2));
            tr("p1+p2");
        }

        /* ================= stage 2 (as[set]): clock-recovery lanes, every lane speculative ================= */
        K2aParams ka[WMB_N_CHAINS];
        const uint32_t Ca = coop ? pick_chunk_coop(c, M) : C;
        const uint32_t lanes_a = (uint32_t)((M + Ca - 1) / Ca);
        /* the two chains' lanes side by side when three threads share a lane: one such warp leaves its scheduler half
         * idle, a second one from the other chain fills it.  (The per-thread kernel keeps its scheduler busier: side by
         * side it was slower.) */
        const bool side = coop && c->chains == 3u;
        CUDA_TRY(cudaStreamWaitEvent(sa, c->ev_k1[set], 0));
        if (side) CUDA_TRY(cudaStreamWaitEvent(c->as2[set], c->ev_k1[set], 0));
        CUDA_TRY(cudaEventRecord(evt[4], sa));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(c->chains & (1u << ch))) continue;
            ChainBuf &b = c->cb[ch];
            SetBuf &sb = b.set[set];
            K2aParams &p = ka[ch];
            memset(&p, 0, sizeof(p));
            p.dphi = sb.dphi + c->W; p.M = M; p.hist = c->hist_m; p.C = Ca; p.W = c->W_a[ch]; p.lanes = lanes_a;
            p.dbits = sb.dbits + wofs; p.sbits = sb.sbits + wofs;
            p.cbits = sb.cbits ? sb.cbits + wofs : nullptr;
            p.st_start = sb.ia_start; p.st_end = sb.ia_end; p.carry = b.ia_carry; p.rerun = sb.rerun_a;
            p.dc = c->o.remove_dc; p.t2 = c->o.t2_enabled; p.lock = c->lock[ch];
            p.mode = 0;
            p.spec0 = first ? 0u : 1u;                   /* the previous batch's lanes may still be running */
            c->st.lanes_run += lanes_a;
            TRY(launch_k2a_lanes(c, ch, p, (side && ch == 0) ? c->as2[set] : sa));     /* S1's lanes are the longer ones: timers on theirs */
        }
        if (side) {
            CUDA_TRY(cudaEventRecord(c->ev_k2a2[set], c->as2[set]));
            CUDA_TRY(cudaStreamWaitEvent(sa, c->ev_k2a2[set], 0));
        }
        CUDA_TRY(cudaEventRecord(evt[5], sa));
        CUDA_TRY(cudaEventRecord(c->ev_k2a[set], sa));
        tr("k1+k2a");

        /* ================= stage 3 (cs): in order from batch to batch ================= */
        CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_k2a[set], 0));
        CUDA_TRY(cudaEventRecord(evt[2], c->cs));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(c->chains & (1u << ch))) continue;
            ChainBuf &b = c->cb[ch];
            TRY(launch_k2a_verify(c, ch, ka[ch]));
            CUDA_TRY(cudaMemcpyAsync(b.ia_carry, b.set[set].ia_end + (ka[ch].lanes - 1), sizeof(IirState), cudaMemcpyDeviceToDevice, c->cs));
            /* the bit history of the run-length warm-ups: the previous batch's last W samples (exact since its fix-up);
             * without -o the demod stream copied the data bits */
            if (!first && c->prev_M % 32 == 0) {         /* only a final (flush) batch can be ragged */
                if (!k1_bits) TRY(copy_history(b.set[set].dbits, b.set[pset].dbits, 4, c->W / 32, c->prev_M / 32, c->cs));
                TRY(copy_history(b.set[set].sbits, b.set[pset].sbits, 4, c->W / 32, c->prev_M / 32, c->cs));
            }
        }

        /* ---- K2t: time2 bit streams straight into the rings (own stream: independent of the
         *      run-length kernels, and both leave most of the GPU idle on their own) ---- */
        if (c->o.t2_enabled) {
            CUDA_TRY(cudaEventRecord(c->ev_fork, c->cs));
            CUDA_TRY(cudaStreamWaitEvent(c->ts, c->ev_fork, 0));
            for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
                if (!(c->chains & (1u << ch))) continue;
                ChainBuf &b = c->cb[ch];
                SetBuf &sb = b.set[set];
                Stream &s = b.s[WMB_ALGO_T2A];
                K2tParams p;
                memset(&p, 0, sizeof(p));
                p.dbits = sb.dbits + wofs; p.sbits = sb.sbits + wofs; p.rssi = sb.rssi + c->W;
                p.M = M; p.lanes = k2t_tiles(M);
                if (p.lanes > c->t2_tiles_max) return set_err(WMB_E_INVAL, "internal: time2 tiles");
                p.cnt = s.cnt; p.tail = b.t2_tail; p.tail_len = b.t2_len; p.base = s.base; p.sr_start = b.t2_sr;
                p.agg_cnt = s.agg; p.agg_tail = b.t2_agg_tail; p.agg_len = b.t2_agg_len;
                p.m_base = (int64_t)c->m_consumed;
                p.ring = s.ring; p.ring_mask = s.ring_cap - 1; p.sd = s.sd; p.cand = s.cand; p.cand_cap = c->cand_cap;
                p.ac_err = c->ac_err[ch];
                TRY(launch_k2t(c, ch, p));
            }
            CUDA_TRY(cudaEventRecord(c->ev_join, c->ts));
        }

        if (early) {
            CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_join_rs, 0));
            CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_join2, 0));
        } else if (c->o.rla_enabled) {
            /* on cs, behind the verification; S1 beside the two-phase path of T1/C1 on s2 (forked after whatever cs
             * holds, joined at the end) */
            const bool s1_beside = (c->chains & 1u) && c->two_phase && (c->chains & 2u);
            if (s1_beside) {
                CUDA_TRY(cudaEventRecord(c->ev_fork2, c->cs));
                CUDA_TRY(cudaStreamWaitEvent(c->s2, c->ev_fork2, 0));
            }
            TRY(enqueue_run_length(c->cs, s1_beside ? c->s2 : c->cs));
            if (s1_beside) {
                CUDA_TRY(cudaEventRecord(c->ev_join2, c->s2));
                CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_join2, 0));
            }
            tr("k2t+p1+p2");
        }
        if (c->o.t2_enabled) CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_join, 0));
        CUDA_TRY(cudaEventRecord(evt[3], c->cs));
    } else {
        CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_k1[set], 0));
        CUDA_TRY(cudaEventRecord(evt[2], c->cs));
        CUDA_TRY(cudaEventRecord(evt[3], c->cs));
    }

    c->last_hist = c->hist_m;
    c->hist_m = std::min<int64_t>(c->hist_m + M, c->W);
    c->iq_consumed += (uint64_t)n_iq;
    c->m_consumed += (uint64_t)M;
    c->st.input_samples += (uint64_t)n_iq;
    c->st.decimated_samples += (uint64_t)M;
    c->st.batches++;
    c->batch_no++;
    c->prev_M = M; c->last_M = M; c->last_set = set;
    c->last_src = src; c->last_bytes = nbytes;
    return WMB_OK;
}

static int consume_oldest(wmb_ctx *c);

/* the carrier a chain listens to, relative to the capture's centre frequency (the mixer of run_batch) */
static double chain_carrier_hz(const wmb_ctx *c, int chain)
{
    if (c->o.simultaneous == 2) return 25e3 * (double)c->o.carrier_25khz[chain];
    if (c->o.simultaneous) return chain == 0 ? 325e3 : -325e3;
    return 0.0;
}

/* one slot's kept granules (fetched whole) -> the granule store; those beyond the slot's pool are lost */
static void book_granules(wmb_ctx *c, const wmb_ctx::InFlight &f, uint64_t n, uint64_t stored)
{
    const uint64_t gb = 4096ull * c->d;
    const uint32_t *list = c->snlist.h + c->snlist.at(f.slot);
    const uint8_t *pool = c->snpool.h + c->snpool.at(f.slot);
    for (uint64_t i = 0; i < n; i++) {
        wmb_ctx::SnipGran &g = c->sn_store[f.sn_g0 + list[i]];
        g.lost = i >= stored;
        if (g.lost) { g.bytes.clear(); continue; }
        const uint64_t at = (uint64_t)list[i] * gb;
        g.bytes.assign(pool + i * gb, pool + i * gb + std::min(gb, f.sn_bytes - at));
    }
    c->st.d2h_bytes += sizeof(uint64_t) + std::max<uint64_t>(n, f.snlist) * sizeof(uint32_t) + std::max<uint64_t>(stored * gb, f.snpool);
}

/* the granules of a piece's snippet: [max(g_first, floor(s / 2048) - PRE), ceil(e / 2048) + POST), the end clipped to
 * the input consumed */
static uint64_t snip_lo(const wmb_ctx *c, uint64_t s)
{
    const uint64_t g = s / WMB_SNIP_GRAN;
    return std::max<uint64_t>(c->sn_g_first, g >= WMB_SNIP_PRE ? g - WMB_SNIP_PRE : 0);
}
static uint64_t snip_hi(uint64_t e) { return (e + WMB_SNIP_GRAN - 1) / WMB_SNIP_GRAN + WMB_SNIP_POST; }

/* drop the granules and matches that no piece still queued or still to come (they start at the burst frontier or
 * later) can need */
static void snip_prune(wmb_ctx *c)
{
    uint64_t s_min = c->burst_frontier;
    for (const wmb_snippet &q : c->sn_queue) s_min = std::min<uint64_t>(s_min, q.start_sample);
    c->sn_store.erase(c->sn_store.begin(), c->sn_store.lower_bound(snip_lo(c, s_min)));
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) c->sn_ok[ch].erase(c->sn_ok[ch].begin(), c->sn_ok[ch].lower_bound(s_min));
}

/* one slot's burst records (fetched whole) -> the queue; the frontier: where the next piece of any chain may start */
static void book_bursts(wmb_ctx *c, const wmb_ctx::InFlight &f)
{
    const BurstSlot bs = c->h_bslot[f.slot];
    uint64_t frontier = f.m_end;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!c->burst_level[ch] || !(c->chains & (1u << ch))) continue;
        const uint32_t n = bs.n[ch];
        const size_t at = c->brec.at(f.slot, ch);
        c->st.d2h_bytes += (uint64_t)std::max(n, f.brec) * sizeof(BurstRec);
        if (f.bqual) c->st.d2h_bytes += (uint64_t)std::max(n, f.bqual) * sizeof(QualAcc);
        for (uint32_t i = 0; i < n; i++) {
            const BurstRec &r = c->brec.h[at + i];
            QueuedBurst qb;
            wmb_burst &b = qb.b;
            memset(&b, 0, sizeof(b));
            if (f.bqual) qb.q = c->bqual.h[at + i]; else qual_zero(qb.q);
            b.start_sample = r.start; b.end_sample = r.end; b.rssi_sum = r.rssi_sum; b.sum = r.sum; b.n = r.n;
            b.chain = r.chain; b.peak = r.peak; b.flags = r.flags;
            /* -a: the cross-product discriminator is not a frequency */
            b.valid = (uint8_t)(r.n > 0 && c->o.accurate_atan ? 1 : 0);
            b.carrier_hz = chain_carrier_hz(c, ch);
            b.offset_hz = b.valid ? (double)r.sum / (double)r.n / (double)WMB_OFS_SCALE * 400e3 / c->fir_gain[ch] : NAN;
            c->bursts.push_back(qb);
            if (c->snip_mode) {
                wmb_snippet sn;
                memset(&sn, 0, sizeof(sn));
                sn.start_sample = r.start; sn.end_sample = r.end; sn.chain = r.chain; sn.flags = r.flags;
                c->sn_queue.push_back(sn);
            }
        }
        if (bs.open[ch] && (uint64_t)bs.ps[ch] < frontier) frontier = (uint64_t)bs.ps[ch];
    }
    c->st.d2h_bytes += sizeof(BurstSlot);
    c->burst_frontier = frontier;
}

/* Enqueue the frame gather (K3), the device framer (K4) and the copies of their results into the host mirror of the
 * next result slot, for everything the streams hold: the candidates carried over plus the new access-code matches.
 * after_batch: this gather closes the batch just enqueued (its set may be reused once it is done).  final: end of
 * input, nothing is carried over. */
static int enqueue_gather(wmb_ctx *c, bool final, bool after_batch)
{
    if (!c->allocated) return WMB_OK;
    const bool any_sync = c->o.rla_enabled || c->o.t2_enabled;
    if (c->inflight.size() >= WMB_NSLOT) TRY(consume_oldest(c));          /* the slot's host mirror must be free */
    const int slot = (int)(c->gather_no % WMB_NSLOT);
    wmb_ctx::InFlight f{};
    const bool quality = c->quality && !c->manual;  /* (a caller's frames carry no sums: manual mode takes none) */
    const bool bursts = bursts_on(c) && (after_batch || final);
    if (bursts) TRY(burst_alloc(c));
    const bool snips = c->snip_mode && bursts && after_batch;
    if (snips) TRY(snip_alloc(c));
    if (quality) TRY(qual_alloc(c));
    const bool repair = c->repair_e && !c->manual;
    const bool repair_soft = repair && (c->repair_k || c->repair_s || c->repair_s1);   /* K4S behind K4R */
    const bool soft_s1 = c->soft_s1 || (repair && c->repair_s1);        /* the S1 streams' values too */
    const bool soft = c->soft || soft_s1 || repair_soft;
    if (repair && !c->rep.d) TRY(c->rep.alloc(c, 1, c->hdr.cap, c->hdr.prefix, 256));     /* first gather with repair on */
    if (soft) TRY(soft_alloc(c, soft_s1));
    if (any_sync) {
        K3Params p;
        memset(&p, 0, sizeof(p));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(c->chains & (1u << ch))) continue;
            for (int a = 0; a < WMB_N_ALGOS; a++) {
                if ((a == WMB_ALGO_RLA && !c->o.rla_enabled) || (a == WMB_ALGO_T2A && !c->o.t2_enabled)) continue;
                Stream &s = c->cb[ch].s[a];
                const int k = ch * WMB_N_ALGOS + a;
                p.ring[k] = s.ring; p.ring_mask[k] = s.ring_cap - 1; p.sd[k] = s.sd; p.cand[k] = s.cand; p.pend[k] = s.pend;
                p.pend_ofs[k] = s.pend_ofs;
                if (quality) p.pend_qual[k] = s.pend_qual;
                if (soft && (ch != WMB_CHAIN_S1 || soft_s1)) p.soft_ring[k] = s.soft_ring;
            }
            p.dphi[ch] = c->cb[ch].set[c->last_set].dphi;
        }
        p.pend_cap = c->pend_cap; p.cand_cap = c->cand_cap;
        /* new matches are those of the batch just enqueued (a gather that closes no batch has none); k3_fill reads their
         * carrier-offset windows from its dphi set */
        p.m_first = (c->m_consumed - (uint64_t)c->last_M) & EVG_M_MASK;
        p.prefix = c->W; p.clip = (uint32_t)c->last_hist; p.batch_m = after_batch ? (uint32_t)c->last_M : 0u;
        p.gd = c->d_gd; p.rec = c->d_rec + slot;
        p.hdr_log = c->hdr.d; p.dec_log = c->dec.d; p.log_base = (uint32_t)c->hdr.at(slot); p.log_cap = (uint32_t)c->hdr.cap;
        p.words = c->d_words; p.words_cap = c->frame_words_cap;
        p.cut_n = c->d_cut_n; p.agg = c->d_k3_agg; p.errors = c->d_errors;
        p.final = final ? 1u : 0u;
        if (quality) { p.qual_log = c->qual.d; p.qual_skip = c->o.accurate_atan ? 0u : 1u; }
        if (soft) p.soft_words = c->d_soft_words;
        K4Params q;
        memset(&q, 0, sizeof(q));
        q.hdr = c->hdr.d; q.words = c->d_words; q.dec = c->dec.d;
        q.pool = c->pool.d + c->pool.at(slot); q.pool_cap = (uint32_t)c->pool.cap; q.pool_n = GD_FIELD(c, pool_n); q.errors = c->d_errors; q.gd = c->d_gd;
        K4RParams r;
        memset(&r, 0, sizeof(r));
        r.hdr = q.hdr; r.dec = q.dec; r.words = q.words; r.rep = c->rep.d; r.pool = q.pool; r.pool_cap = q.pool_cap;
        r.pool_n = q.pool_n; r.errors = q.errors; r.e_max = c->repair_e; r.gd = q.gd;
        K4SParams sp;
        memset(&sp, 0, sizeof(sp));
        sp.hdr = r.hdr; sp.dec = r.dec; sp.words = r.words; sp.soft = c->d_soft_words; sp.rep = r.rep; sp.pool = r.pool;
        sp.pool_cap = r.pool_cap; sp.pool_n = r.pool_n; sp.errors = r.errors; sp.k_max = c->repair_k; sp.s_max = c->repair_s;
        sp.s1_max = c->repair_s1; sp.gd = r.gd;
        TRY(launch_k3_k4(c, p, c->manual ? nullptr : &q, repair ? &r : nullptr, repair_soft ? &sp : nullptr));
        /* results -> pinned host mirror: the record and a prefix of the arrays it describes (the rest, if a batch ever
         * produces more, is fetched when the record has been read) */
        CUDA_TRY(cudaMemcpyAsync(c->h_rec + slot, c->d_rec + slot, sizeof(BatchRec), cudaMemcpyDeviceToHost, c->cs));
        TRY(c->hdr.enqueue(slot, 0, c->cs, &f.hdr));
        if (quality) TRY(c->qual.enqueue(slot, 0, c->cs, &f.qual));
        if (!c->manual) {
            TRY(c->dec.enqueue(slot, 0, c->cs, &f.dec));
            TRY(c->pool.enqueue(slot, 0, c->cs, &f.pool));
            if (repair) TRY(c->rep.enqueue(slot, 0, c->cs, &f.rep));
        }
    }
    /* the burst report: behind the demod kernel of the batch (cs waited for it), before ev_chain[set] releases the set */
    const bool bqual = bursts && c->quality;
    if (bursts) {
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!c->burst_level[ch] || !(c->chains & (1u << ch))) continue;
            const wmb_ctx::BurstBuf &b = c->bb[ch];
            BurstParams p;
            memset(&p, 0, sizeof(p));
            const SetBuf &sb = c->cb[ch].set[c->last_set];
            /* batch sample 0 = decimated sample m_first; the end-of-input gather (M = 0) comes after the last batch, whose
             * set ends at m_first: the quality pass may read the window of a piece closed there out of that set */
            p.rssi = sb.rssi + c->W; p.dphi = sb.dphi + c->W + (after_batch ? 0 : c->last_M);
            p.M = after_batch ? c->last_M : 0;
            p.clip = c->last_hist;
            p.m_first = (int64_t)(c->m_consumed - (uint64_t)p.M);
            p.level = c->burst_level[ch]; p.chain = (uint32_t)ch; p.final_ = final ? 1u : 0u;
            p.nw = (uint32_t)((p.M + 31) / 32); p.units = (uint32_t)((p.M + WMB_BURST_UNIT - 1) / WMB_BURST_UNIT);
            p.mask = b.mask; p.cnt = b.cnt; p.base = b.base; p.ev = b.ev; p.bd = b.bd; p.items = b.items;
            p.out = c->brec.d + c->brec.at(slot, ch);
            p.slot = c->d_bslot + slot;
            if (bqual) {
                p.qout = c->bqual.d + c->bqual.at(slot, ch);
                p.qual_skip = c->o.accurate_atan ? 0u : 1u;
            }
            TRY(launch_bursts(c, p, b.agg));
        }
        CUDA_TRY(cudaMemcpyAsync(c->h_bslot + slot, c->d_bslot + slot, sizeof(BurstSlot), cudaMemcpyDeviceToHost, c->cs));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!c->burst_level[ch] || !(c->chains & (1u << ch))) continue;
            TRY(c->brec.enqueue(slot, ch, c->cs, &f.brec));
            if (bqual) TRY(c->bqual.enqueue(slot, ch, c->cs, &f.bqual));
        }
    }
    /* the snippet pass: behind kb_mask of the burst-on chains, on the batch's input bytes.  A host push's next H2D into
     * the same input buffer waits for ev_snip; a device push returns only after consume_all, so the caller's buffer is
     * read before it may be reused */
    if (snips) {
        SnipParams p;
        memset(&p, 0, sizeof(p));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++)
            if (c->burst_level[ch] && (c->chains & (1u << ch))) p.mask[ch] = c->bb[ch].mask;
        const uint64_t m_first = c->m_consumed - (uint64_t)c->last_M;
        p.nw = (uint32_t)((c->last_M + 31) / 32);
        p.ng = (uint32_t)((c->last_M + WMB_SNIP_GRAN - 1) / WMB_SNIP_GRAN);
        p.g0 = m_first / WMB_SNIP_GRAN;
        p.keep = c->d_snkeep; p.rank = c->d_snrank; p.sd = c->d_snd;
        p.in = c->last_src; p.in_bytes = c->last_bytes; p.gbytes = 4096u * c->d;
        p.pool_gran = c->snip_pool_gran;
        p.pool = c->snpool.d + c->snpool.at(slot); p.list = c->snlist.d + c->snlist.at(slot);
        TRY(launch_snippets(c, p, c->d_snn + slot));
        for (int i = 0; i < 2; i++)
            if (c->last_src == c->d_in[i]) CUDA_TRY(cudaEventRecord(c->ev_snip[i], c->cs));
        CUDA_TRY(cudaMemcpyAsync(c->h_snn + slot, c->d_snn + slot, sizeof(uint64_t), cudaMemcpyDeviceToHost, c->cs));
        TRY(c->snlist.enqueue(slot, 0, c->cs, &f.snlist));
        TRY(c->snpool.enqueue(slot, 0, c->cs, &f.snpool));
        f.sn = true; f.sn_g0 = p.g0; f.sn_bytes = c->last_bytes;
    }
    /* the band survey: the rows the batch closed (its kernels ran on the demod stream), or at the end of input the
     * record still open */
    if (c->spec_bins) {
        std::vector<wmb_spectrum_row> &rows = c->spec_slot_rows[slot];
        rows.clear();
        /* cs follows the demod stream only as far as the demod kernel; the survey kernels behind it may still be adding
         * into the open record's ring row.  Every close that cs issues (the flush's, or the next solo batch's on sk = cs)
         * and every copy of a slot comes after this wait, whether the batch closed a record or not */
        if (c->spec_enqueued) {
            CUDA_TRY(cudaStreamWaitEvent(c->cs, c->ev_spec, 0));
            c->spec_enqueued = false;
        }
        if (after_batch && !c->spec_batch_rows.empty()) {
            rows.swap(c->spec_batch_rows);
        } else if (final && c->spec_open >= 0) {
            rows.push_back(spec_row(c, c->spec_open, c->spec_open_blocks));
            SpecCloseParams q;
            memset(&q, 0, sizeof(q));
            q.sum = c->d_ssum_ring; q.peak = c->d_speak_ring;
            q.out_sum = c->ssum.d + c->ssum.at(slot); q.out_peak = c->speak.d + c->speak.at(slot);
            q.lone = c->spec_open; q.n = 1; q.N = c->spec_bins; q.R = c->spec_R;
            TRY(launch_spec_close(c, q, c->cs));
            CUDA_TRY(cudaEventRecord(c->ev_spec_flush, c->cs));
            c->spec_flush_pending = true;
            c->spec_open = -1; c->spec_open_blocks = 0;
        }
        if (!rows.empty()) {
            c->ssum.prefix = c->speak.prefix = (uint32_t)rows.size() * c->spec_bins;     /* exact */
            TRY(c->ssum.enqueue(slot, 0, c->cs, &f.ssum));
            TRY(c->speak.enqueue(slot, 0, c->cs, &f.speak));
        }
    }
    CUDA_TRY(cudaEventRecord(c->ev_res[slot], c->cs));
    /* ev_chain[set] releases the batch's set to the demod kernel of batch i+2 (run_batch waits for it on k1s): it is
     * recorded here, behind the gather on cs, so k3_fill's reads of the set's dphi come before that kernel's writes */
    if (after_batch) {
        CUDA_TRY(cudaEventRecord(c->ev_chain[c->last_set], c->cs));
        c->chain_recorded[c->last_set] = true;
    }
    f.slot = slot; f.final = final; f.has_timers = after_batch; f.m_end = c->m_consumed; f.iq_end = c->iq_consumed;
    c->inflight.push_back(f);
    c->gather_no++;
    return WMB_OK;
}

static int book_device_frames(wmb_ctx *c, const FrameHdr *hdr, const DecHdr *dec, const QualAcc *qual, const RepHdr *rep,
                              const uint8_t *pool, size_t n, bool final);

/* Wait for the oldest gathered batch's results (an event, not a stream: later batches keep running), fetch what the
 * prefix copy did not cover, and run the stream-order bookkeeping over it. */
static int consume_oldest(wmb_ctx *c)
{
    if (c->inflight.empty()) return WMB_OK;
    const wmb_ctx::InFlight f = c->inflight.front();
    c->inflight.erase(c->inflight.begin());
    const double t0 = wall_ms();
    CUDA_TRY(cudaEventSynchronize(c->ev_res[f.slot]));
    const double t1 = wall_ms();
    c->st.host_gather_ms += t1 - t0;
    if (f.has_timers) {
        float ms = 0.f;
        cudaEvent_t *evt = c->ev_t[f.slot];
        const bool any = c->o.rla_enabled || c->o.t2_enabled;
        if (cudaEventElapsedTime(&ms, evt[0], evt[1]) == cudaSuccess) c->acc_demod_ms += ms;
        if (any && cudaEventElapsedTime(&ms, evt[4], evt[5]) == cudaSuccess) c->acc_bitsync_ms += ms;     /* clock-recovery lanes */
        if (cudaEventElapsedTime(&ms, evt[2], evt[3]) == cudaSuccess) c->acc_bitsync_ms += ms;            /* bit streams */
        /* the whole per-sample pass of the push so far: first demod kernel -> this batch's last bit-sync kernel */
        if (cudaEventElapsedTime(&ms, c->ev_push_start, evt[3]) == cudaSuccess) c->acc_pass_ms = ms;
    }
    /* what the prefix copies missed, on xs, and one wait for all of it: the slot is not written again before it is read */
    const BatchRec r = f.hdr ? c->h_rec[f.slot] : BatchRec{};
    uint32_t most = 0;                               /* burst records of the slot's fullest chain */
    bool more = false;
    for (int ch = 0; f.brec && ch < WMB_N_CHAINS; ch++) {
        if (!c->burst_level[ch] || !(c->chains & (1u << ch))) continue;
        const uint32_t n = c->h_bslot[f.slot].n[ch];
        TRY(c->brec.fetch(f.slot, ch, f.brec, n, c->xs, &more));
        if (f.bqual) TRY(c->bqual.fetch(f.slot, ch, f.bqual, n, c->xs, &more));
        most = std::max(most, n);
    }
    const uint64_t sn_n = f.sn ? c->h_snn[f.slot] : 0;                   /* granules the batch kept */
    const uint64_t sn_stored = std::min<uint64_t>(sn_n, c->snip_pool_gran);
    const uint32_t gbytes = 4096u * c->d;
    if (f.sn) {
        TRY(c->snlist.fetch(f.slot, 0, f.snlist, (uint32_t)sn_n, c->xs, &more));
        TRY(c->snpool.fetch(f.slot, 0, f.snpool, (uint32_t)(sn_stored * gbytes), c->xs, &more));
    }
    TRY(c->hdr.fetch(f.slot, 0, f.hdr, r.n, c->xs, &more));
    if (f.dec) TRY(c->dec.fetch(f.slot, 0, f.dec, r.n, c->xs, &more));
    if (f.qual) TRY(c->qual.fetch(f.slot, 0, f.qual, r.n, c->xs, &more));
    if (f.pool) TRY(c->pool.fetch(f.slot, 0, f.pool, r.pool_n, c->xs, &more));
    if (f.rep) TRY(c->rep.fetch(f.slot, 0, f.rep, r.n, c->xs, &more));
    if (!f.dec && r.n_words) {               /* manual mode reads after every batch: the frame words are this batch's */
        CUDA_TRY(cudaMemcpyAsync(c->h_words, c->d_words, (size_t)r.n_words * 4, cudaMemcpyDeviceToHost, c->xs));
        c->st.d2h_bytes += (uint64_t)r.n_words * 4;
        if (c->soft || c->soft_s1) {
            CUDA_TRY(cudaMemcpyAsync(c->h_soft_words, c->d_soft_words, (size_t)r.n_words * 2, cudaMemcpyDeviceToHost, c->xs));
            c->st.d2h_bytes += (uint64_t)r.n_words * 2;
        }
        more = true;
    }
    if (more) CUDA_TRY(cudaStreamSynchronize(c->xs));
    /* the next batches probably look like this one: let the prefix copies cover them */
    if (f.brec) { c->brec.grow(most); c->bqual.grow(most); }
    if (f.hdr) { c->hdr.grow(r.n); c->dec.grow(r.n); c->qual.grow(r.n); c->rep.grow(r.n); c->pool.grow(r.pool_n); }
    if (f.sn) {
        c->snlist.grow((uint32_t)sn_n); c->snpool.grow((uint32_t)(sn_stored * gbytes));
        book_granules(c, f, sn_n, sn_stored);
    }
    if (f.final) c->flushed = true;
    c->sn_iq_end = f.iq_end;
    if (f.brec) book_bursts(c, f);
    if (c->snip_mode) snip_prune(c);
    if (f.ssum) {                                    /* the slot's survey rows -> the queue */
        const std::vector<wmb_spectrum_row> &rows = c->spec_slot_rows[f.slot];
        const size_t at = c->ssum.at(f.slot);        /* = c->speak.at(f.slot): both hold rows x bins */
        c->spec_rows.insert(c->spec_rows.end(), rows.begin(), rows.end());
        c->spec_sum.insert(c->spec_sum.end(), c->ssum.h + at, c->ssum.h + at + f.ssum);
        c->spec_peak.insert(c->spec_peak.end(), c->speak.h + at, c->speak.h + at + f.speak);
        c->st.d2h_bytes += (uint64_t)f.ssum * sizeof(uint64_t) + (uint64_t)f.speak * sizeof(uint32_t);
    }
    if (!f.hdr) {
        if (sn_n > sn_stored) c->st.overflow_batches++;
        return WMB_OK;
    }
    const uint32_t err = r.errors;
    if (err & 2u) return set_err(WMB_E_OVERFLOW, "run-length tracker left its defined range (the reference would spin here)");
    /* lane event buffer (1: a run-length lane emitted more than one bit per four samples plus one capped edge -- the
     * tracker's bit length has collapsed to a fraction of a sample), frame words (4), datagram pool (8), access-code
     * matches (16), pending candidates (64): the device dropped what did not fit and cleared the flags; the reference
     * would have gone on decoding, so does the stream */
    if ((err & K3_SOFT_ERRORS) || sn_n > sn_stored) c->st.overflow_batches++;
    if (err & 256u) return set_err(WMB_E_STATE, "internal: lane verification does not converge");
    c->st.d2h_bytes += sizeof(BatchRec) + (size_t)r.n * sizeof(FrameHdr) + (f.dec ? (size_t)r.n * sizeof(DecHdr) + r.pool_n : 0);
    if (f.qual) c->st.d2h_bytes += (size_t)r.n * sizeof(QualAcc);
    if (f.rep) c->st.d2h_bytes += (size_t)r.n * sizeof(RepHdr);
    /* statistics kept on the device */
    c->st.lanes_rerun += r.lanes_rerun - c->stat_rerun_seen; c->st.lanes_run += r.lanes_rerun - c->stat_rerun_seen;
    c->stat_rerun_seen = r.lanes_rerun;
    c->st.rl_fallbacks += r.rl_fallbacks - c->stat_fallback_seen;
    c->stat_fallback_seen = r.rl_fallbacks;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++)
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            const int k = ch * WMB_N_ALGOS + a;
            c->st.candidates[ch][a] = r.n_cand_total[k];
            /* stage tap: the events of the batch this gather closes (has_timers).  Records are read in batch order, so
             * the total before it is the one the record before read -- not s.total when the batch was enqueued, which
             * lags by the batches still in flight then */
            if (f.has_timers) c->cb[ch].s[a].total_prev = c->cb[ch].s[a].total;
            c->cb[ch].s[a].total = r.total[k];
        }
    FrameHdr *hdr = c->hdr.h + c->hdr.at(f.slot);
    /* the device keeps 40 bits of the sample index; widen to the 64-bit stream position: the newest value
     * congruent to it that is not beyond the samples produced when the batch was gathered */
    for (uint32_t i = 0; i < r.n; i++) hdr[i].sync_sample = f.m_end - ((f.m_end - hdr[i].sync_sample) & EVG_M_MASK);
    int rc = WMB_OK;
    if (f.dec) rc = book_device_frames(c, hdr, c->dec.h + c->dec.at(f.slot), f.qual ? c->qual.h + c->qual.at(f.slot) : nullptr,
                                       f.rep ? c->rep.h + c->rep.at(f.slot) : nullptr, c->pool.h + c->pool.at(f.slot), r.n, f.final);
    else {
        /* manual mode: keep the frames (newest version of a re-delivered partial one wins) for wmb_poll */
        for (uint32_t i = 0; i < r.n; i++) {
            const FrameHdr &h = hdr[i];
            if (h.nbits == 0) continue;
            wmb_frame fr;
            memset(&fr, 0, sizeof(fr));
            fr.sync_sample = h.sync_sample; fr.ordinal = h.ordinal; fr.chain = h.chain; fr.algo = h.algo;
            fr.truncated = (uint8_t)((h.complete && !h.cut) ? 0 : 1);
            fr.reserved = (uint8_t)((!h.complete && !f.final) ? 1 : 0);      /* partial: will be re-delivered */
            fr.nbits = h.nbits;
            wmb_ctx::Held *slot = nullptr;
            for (auto &hh : c->held)
                if (hh.f.chain == fr.chain && hh.f.algo == fr.algo && hh.f.ordinal == fr.ordinal) { slot = &hh; break; }
            if (!slot) { c->held.emplace_back(); slot = &c->held.back(); }
            slot->f = fr;
            slot->words.assign(c->h_words + h.word_off, c->h_words + h.word_off + h.nbits);
            if (h.chain == WMB_CHAIN_T1C1 ? c->soft : c->soft_s1) slot->soft.assign(c->h_soft_words + h.word_off, c->h_soft_words + h.word_off + h.nbits);
            else slot->soft.clear();
        }
    }
    c->st.host_decode_ms += wall_ms() - t1;
    return rc;
}

static int consume_all(wmb_ctx *c)
{
    while (!c->inflight.empty()) TRY(consume_oldest(c));
    c->st.demod_kernel_ms = c->acc_demod_ms; c->st.bitsync_kernel_ms = c->acc_bitsync_ms; c->st.batch_device_ms = c->acc_pass_ms;
    tr("consumed");
    tr_dump();
    return WMB_OK;
}

/* --------------------------------------------------------------------------- */
/* push / poll                                                                 */
/* --------------------------------------------------------------------------- */

static int process_device_batches(wmb_ctx *c, const uint8_t *dev, size_t nbytes, bool final);

static double wall_ms()
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec;
}

/* gather what the batch just enqueued produced; manual mode reads it at once (the frame words are per batch) */
static int finish_batch(wmb_ctx *c, bool final, bool after_batch)
{
    TRY(enqueue_gather(c, final, after_batch));
    if (c->manual) TRY(consume_all(c));
    return WMB_OK;
}

static size_t batch_granule(const wmb_ctx *c) { return (size_t)4096 * c->d; }

extern "C" int wmb_push_device(wmb_ctx *c, const void *dev_cu8, size_t nbytes)
{
    if (!c || (!dev_cu8 && nbytes)) return set_err(WMB_E_INVAL, "null argument");
    if (nbytes % 4096) return set_err(WMB_E_INVAL, "wmb_push_device needs a multiple of 4096 bytes");
    if (((uintptr_t)dev_cu8) & 15u) return set_err(WMB_E_INVAL, "device buffer must be 16-byte aligned");
    if (!c->remainder.empty()) return set_err(WMB_E_STATE, "wmb_push_device after a partial push");
    CUDA_TRY(cudaSetDevice(c->device));
    int rc = ctx_alloc(c);
    if (rc) return rc;
    /* whole decimation granules (4096 * d bytes) go to the device as they are; a trailing partial granule (a capture
     * whose length is a multiple of 4096 but not of 4096 * d) waits on the host side like the remainder of a host push */
    const size_t tail = nbytes % batch_granule(c);
    rc = process_device_batches(c, (const uint8_t *)dev_cu8, nbytes - tail, false);
    if (rc) return rc;
    rc = consume_all(c);                                  /* also: the caller's buffer is no longer in use (the snippet copy reads it) */
    if (rc || !tail) return rc;
    c->remainder.resize(tail);
    CUDA_TRY(cudaMemcpy(c->remainder.data(), (const uint8_t *)dev_cu8 + (nbytes - tail), tail, cudaMemcpyDeviceToHost));
    return WMB_OK;
}

/* dev points to device memory that stays valid until the results have been consumed.  A long push is cut into
 * batches that follow each other through the device like through a pipeline: the demod kernel of batch i+1 runs
 * beside the latency-bound bit-stream kernels of batch i (run_batch), and the host books batch i's results while
 * later batches are still running. */
static int process_device_batches(wmb_ctx *c, const uint8_t *dev, size_t nbytes, bool final)
{
    const size_t gran = batch_granule(c);
    size_t cap = std::min(c->max_batch_bytes, g_pipe_bytes);
    cap -= cap % gran;
    if (!cap) cap = gran;
    size_t off = 0;
    c->acc_demod_ms = c->acc_bitsync_ms = c->acc_pass_ms = 0; c->push_started = false;
    while (off < nbytes) {
        size_t n = std::min(nbytes - off, cap);
        if (nbytes - off - n < cap / 4) n = nbytes - off;                /* no dwarf batch at the end */
        if (n > c->max_batch_bytes) n = c->max_batch_bytes;
        if (n < nbytes - off || !final) {
            /* keep batch boundaries on whole decimation periods */
            if (n % gran) n -= n % gran;
            if (n == 0) break;
        }
        const double tb = wall_ms();
        int rc = run_batch(c, dev + off, n, nullptr, off + n >= nbytes);
        if (rc) return rc;
        c->st.host_batch_ms += wall_ms() - tb;
        rc = finish_batch(c, false, true);
        if (rc) return rc;
        off += n;
    }
    if (off < nbytes) return set_err(WMB_E_INVAL, "device push must be a multiple of %zu bytes unless flushing", gran);
    return WMB_OK;
}

/* host bytes -> device (double-buffered) -> batches */
static int push_host_bytes(wmb_ctx *c, const uint8_t *p, size_t nbytes, bool final)
{
    const size_t gran = batch_granule(c);
    size_t off = 0;
    /* enqueue the first H2D, then for each batch: enqueue the next H2D before computing */
    size_t cur_n = 0;
    /* Batch sizes: the maximum while plenty is left, then a taper (7/16 of what is left, not below half a
     * batch): the copy of batch i+1 hides behind the kernels of batch i, so what a caller waits for after the
     * last byte has crossed PCIe is the LAST batch's kernels -- a smaller last batch shortens that, as long as
     * every batch still computes faster than the next one copies (the lane warm-ups are a fixed cost per batch,
     * the copy grows with its size). */
    auto next_size = [&](size_t at) {
        const size_t rem = nbytes - at, mx = c->max_batch_bytes, half = mx / 2;
        size_t n;
        if (rem > 2 * mx) n = mx;
        else if (rem <= half + half / 2) n = rem;
        else if (rem <= 2 * half) n = rem - half;
        else n = std::min(mx, std::max(half, rem / 16 * 7));
        if (!(final && at + n == nbytes)) n -= n % gran;
        if (n == 0 && rem >= gran) n = gran;
        return n;
    };
    cur_n = next_size(0);
    if (cur_n == 0) {
        c->remainder.assign(p, p + nbytes);             /* less than one granule: keep for later */
        return WMB_OK;
    }
    c->acc_demod_ms = c->acc_bitsync_ms = c->acc_pass_ms = 0; c->push_started = false;
    int idx = c->buf_idx;
    CUDA_TRY(cudaStreamWaitEvent(c->xs, c->ev_k1done[idx], 0));
    if (c->ev_snip[idx]) CUDA_TRY(cudaStreamWaitEvent(c->xs, c->ev_snip[idx], 0));     /* the snippet copy read it */
    CUDA_TRY(cudaMemcpyAsync(c->d_in[idx], p, cur_n, cudaMemcpyHostToDevice, c->xs));
    CUDA_TRY(cudaEventRecord(c->ev_h2d[idx], c->xs));
    while (cur_n) {
        const size_t nxt_off = off + cur_n;
        const size_t nxt_n = nxt_off < nbytes ? next_size(nxt_off) : 0;
        if (nxt_n) {
            const int nidx = idx ^ 1;
            CUDA_TRY(cudaStreamWaitEvent(c->xs, c->ev_k1done[nidx], 0));
            if (c->ev_snip[nidx]) CUDA_TRY(cudaStreamWaitEvent(c->xs, c->ev_snip[nidx], 0));
            CUDA_TRY(cudaMemcpyAsync(c->d_in[nidx], p + nxt_off, nxt_n, cudaMemcpyHostToDevice, c->xs));
            CUDA_TRY(cudaEventRecord(c->ev_h2d[nidx], c->xs));
        }
        c->buf_idx = idx;
        const double tb = wall_ms();
        int rc = run_batch(c, c->d_in[idx], cur_n, c->ev_h2d[idx], nxt_n == 0);
        if (rc) return rc;
        c->st.host_batch_ms += wall_ms() - tb;
        c->st.h2d_bytes += cur_n;
        rc = finish_batch(c, false, true);
        if (rc) return rc;
        off = nxt_off; cur_n = nxt_n; idx ^= 1;
    }
    c->buf_idx = idx;
    CUDA_TRY(cudaStreamSynchronize(c->xs));             /* the caller may reuse its buffer now */
    if (off < nbytes) c->remainder.assign(p + off, p + nbytes);
    return consume_all(c);
}

extern "C" int wmb_push(wmb_ctx *c, const uint8_t *cu8, size_t nbytes)
{
    if (!c || (!cu8 && nbytes)) return set_err(WMB_E_INVAL, "null argument");
    CUDA_TRY(cudaSetDevice(c->device));
    int rc = ctx_alloc(c);
    if (rc) return rc;
    if (!c->remainder.empty()) {
        /* complete the pending granule first (remainder is always shorter than one granule) */
        const size_t gran = batch_granule(c);
        const size_t take = std::min(gran - c->remainder.size(), nbytes);
        c->remainder.insert(c->remainder.end(), cu8, cu8 + take);
        cu8 += take; nbytes -= take;
        if (c->remainder.size() < gran) return WMB_OK;
        std::vector<uint8_t> tmp;
        tmp.swap(c->remainder);
        rc = push_host_bytes(c, tmp.data(), tmp.size(), false);
        if (rc) return rc;
        if (!nbytes) return WMB_OK;
    }
    return push_host_bytes(c, cu8, nbytes, false);
}

/* end of input: process what is left in whole 4096-byte items (rtl_wmbus.c:1301-1308) */
static int flush_input(wmb_ctx *c)
{
    int rc = ctx_alloc(c);
    if (rc) return rc;
    if (!c->remainder.empty()) {
        std::vector<uint8_t> tmp;
        tmp.swap(c->remainder);
        const size_t n = tmp.size() - tmp.size() % 4096;
        if (n) {
            rc = push_host_bytes(c, tmp.data(), n, true);
            if (rc) return rc;
            c->remainder.clear();
        }
    }
    rc = finish_batch(c, true, false);
    if (rc) return rc;
    return consume_all(c);
}

extern "C" int wmb_poll(wmb_ctx *c, wmb_frame *out, size_t cap, size_t *n, int flush)
{
    if (!c || !n) return set_err(WMB_E_INVAL, "null argument");
    *n = 0;
    CUDA_TRY(cudaSetDevice(c->device));
    if (flush) {
        int rc = flush_input(c);
        if (rc) return rc;
    }
    if (out) {
        c->poll_frames.clear();
        for (auto &h : c->held) { h.f.bits = h.words.data(); c->poll_frames.push_back(h.f); }
        const size_t k = std::min(cap, c->poll_frames.size());
        memcpy(out, c->poll_frames.data(), k * sizeof(wmb_frame));
        *n = k;
        /* the words stay valid until the next push/poll; forget the frames themselves */
        c->held_prev.swap(c->held);
        c->held.clear();
    }
    return WMB_OK;
}

/* --------------------------------------------------------------------------- */
/* host framers: stream-order bookkeeping around wmb_frame_decode()            */
/* --------------------------------------------------------------------------- */

/* Stream-order bookkeeping over decoded candidates (sorted by chain, algorithm, ordinal): a decoder
 * that is receiving ignores further access-code matches (t1_c1_packet_decoder.h:272-278 honours the
 * flag only in idle), so a candidate inside the telegram of an earlier one is dropped; the rest
 * become lines, queued in the order the reference prints them.  accepted (if given): the indices of the frames that the rule
 * accepted, in input order. */
struct FrameMeta { uint8_t chain, algo, partial, truncated, ofs_valid; uint64_t ordinal, sync_sample; int64_t ofs_sum; uint32_t ofs_n;
                   const QualAcc *qual; /* null: no quality sums */ };
struct DecLite { int status; uint32_t consumed; uint64_t end_sample; uint8_t crc_ok; };

template <class Meta, class Lite, class Fill>
static int book_frames(wmb_ctx *c, size_t n, Meta meta, Lite lite, Fill fill, std::vector<size_t> *accepted = nullptr)
{
    struct Key { uint64_t end_sample; uint32_t prio, seq; size_t fi; uint8_t algo; };
    bool blocked[WMB_N_CHAINS][WMB_N_ALGOS] = {{false, false}, {false, false}};
    std::vector<Key> fresh;
    for (size_t fi = 0; fi < n; fi++) {
        const FrameMeta f = meta(fi);
        Stream &s = c->cb[f.chain].s[f.algo];
        if (blocked[f.chain][f.algo]) continue;
        if ((int64_t)f.ordinal <= s.busy_until) continue;
        const DecLite d = lite(fi);
        if (d.status == WMB_DEC_NEED_MORE) {
            if (f.partial) { blocked[f.chain][f.algo] = true; continue; }   /* comes again */
            if (!f.truncated) return set_err(WMB_E_STATE, "internal: frame shorter than its header demands");
            /* cut by a run-length reset or by the end of input: the reference's decoder is reset too */
            s.busy_until = (int64_t)(f.ordinal + d.consumed - 1);
            if (accepted) accepted->push_back(fi);
            continue;
        }
        s.busy_until = (int64_t)(f.ordinal + d.consumed - 1);
        if (accepted) accepted->push_back(fi);
        if (d.status == WMB_DEC_LINE && f.sync_sample >= c->win_lo && f.sync_sample < c->win_hi) {
            Key k;
            k.end_sample = d.end_sample;
            k.prio = (uint32_t)(f.chain * 2 + (f.algo == WMB_ALGO_T2A ? 1 : 0));
            k.seq = (uint32_t)fresh.size(); k.fi = fi; k.algo = f.algo;
            fresh.push_back(k);
            c->st.lines[f.chain][f.algo]++;
            if (d.crc_ok) c->st.lines_crc_ok[f.chain][f.algo]++;
            if (d.crc_ok && c->snip_mode) c->sn_ok[f.chain].insert(f.sync_sample);
        }
    }
    /* the reference prints in the order the per-sample state machines finish:
     * sample index, then T1/C1-rla, T1/C1-t2a, S1-rla, S1-t2a (rtl_wmbus.c:1354-1355).
     * Only the small keys are sorted; the datagrams are materialised once, in print order. */
    auto before = [](const Key &a, const Key &b) {
        if (a.end_sample != b.end_sample) return a.end_sample < b.end_sample;
        if (a.prio != b.prio) return a.prio < b.prio;
        return a.seq < b.seq;
    };
    /* the candidates come stream by stream and, inside a stream, in bit order: the accepted ones of a stream do not
     * overlap, so each stream's lines already are in print order -- merge the (at most four) runs instead of sorting
     * (15 k lines per GiB on dense traffic: 1 ms of std::sort) */
    {
        std::vector<size_t> cut(1, 0);
        bool runs_sorted = true;
        for (size_t i = 1; i < fresh.size(); i++) {
            if (fresh[i].prio != fresh[i - 1].prio) cut.push_back(i);
            else if (before(fresh[i], fresh[i - 1])) runs_sorted = false;
        }
        cut.push_back(fresh.size());
        if (!runs_sorted || cut.size() > 6) std::sort(fresh.begin(), fresh.end(), before);
        else
            for (size_t r = 2; r < cut.size(); r++)
                std::inplace_merge(fresh.begin(), fresh.begin() + (long)cut[r - 1], fresh.begin() + (long)cut[r], before);
    }
    const size_t base = c->lines.size();
    c->lines.resize(base + fresh.size());
    for (size_t i = 0; i < fresh.size(); i++) {
        QueuedLine &q = c->lines[base + i];
        q.end_sample = fresh[i].end_sample; q.prio = (int)fresh[i].prio; q.algo = fresh[i].algo;
        const FrameMeta m = meta(fresh[i].fi);
        q.chain = m.chain; q.sync_sample = m.sync_sample;
        q.ofs_valid = m.ofs_valid; q.ofs_sum = m.ofs_sum; q.ofs_n = m.ofs_n;
        if (m.qual) q.qual = *m.qual; else qual_zero(q.qual);
        fill(fresh[i].fi, q.d);
        if (c->telegrams) {
            wmb_line_info r;
            memset(&r, 0, sizeof(r));
            r.sync_sample = q.sync_sample; r.end_sample = q.end_sample;
            r.chain = q.chain; r.algo = q.algo; r.crc_ok = q.d.crc_ok;
            c->tg_info.push_back(r);
            c->tg_line.push_back(q.d);
        }
    }
    return WMB_OK;
}

/* a K4 verdict -> the decoded telegram, its datagram out of the slot's pool (K4_SKIP: a frame without any bit) */
static void decoded_from(const DecHdr &d, uint64_t sync_sample, const uint8_t *pool, wmb_decoded &o)
{
    static const char modes[3][3] = { "T1", "C1", "S1" };
    memset(&o, 0, sizeof(o));
    o.status = d.status == K4_SKIP ? (int)WMB_DEC_NEED_MORE : (int)d.status;
    o.consumed = d.consumed;
    o.end_sample = d.status == K4_SKIP ? 0 : sync_sample + d.end_off;
    if (d.status != K4_LINE) return;
    memcpy(o.mode, modes[d.mode < 3 ? d.mode : 0], 3);
    o.crc_ok = d.crc_ok; o.ok_3of6 = d.ok_3of6; o.packet_rssi = d.packet_rssi; o.current_rssi = d.current_rssi;
    o.serial = d.serial; o.len = d.len;
    memcpy(o.datagram, pool + d.data_off, d.len);
}

/* the mode of a candidate's repaired line: K4R repairs T1 and S1 telegrams, K4S C1 lines (K4's verdict says which) */
static int rep_mode(int chain, const DecHdr &d)
{
    if (chain != WMB_CHAIN_T1C1) return 2;
    return d.status == K4_LINE && d.mode == 1 ? 1 : 0;
}

/* a K4R / K4S verdict -> the repair of one candidate, its datagram out of the pool */
static void repaired_from(const RepHdr &h, uint64_t sync_sample, int mode, const uint8_t *pool, wmb_repaired &o)
{
    static const char modes[3][3] = { "T1", "C1", "S1" };
    memset(&o, 0, sizeof(o));
    o.outcome = h.outcome; o.had_line = h.had_line & 1u;             /* bits 1, 2: K4S's T1 / S1 soft rule decided */
    if (h.outcome != K4R_REPAIRED) return;
    o.erasures = h.erasures; o.blocks = h.blocks;
    wmb_decoded &d = o.line;
    d.status = WMB_DEC_LINE; d.consumed = h.consumed; d.end_sample = sync_sample + h.end_off;
    memcpy(d.mode, modes[mode], 3);
    d.crc_ok = 1; d.ok_3of6 = 1; d.packet_rssi = h.packet_rssi; d.current_rssi = h.current_rssi;
    d.serial = h.serial; d.len = h.len;
    memcpy(d.datagram, pool + h.data_off, h.len);
}

/* The repair records of one gathered batch (wmb_set_repair).  A candidate that book_frames accepted gets its record in
 * the gather that delivers it with all its bits (not partial).  An S1 abort is accepted as soon as K4 sees the
 * violation, usually long before bit P - 1: K3 carries it on, and it waits in its stream's rep_wait list for that
 * gather.  A waiting frame that a gather does not deliver was lost in an overflow (counted there). */
static void book_repairs(wmb_ctx *c, const FrameHdr *hdr, const DecHdr *dec, const RepHdr *rep, const uint8_t *pool, size_t n,
                         const std::vector<uint32_t> &idx, const std::vector<size_t> &accepted, bool final)
{
    std::vector<wmb_repair_record> fresh;
    auto partial = [&](uint32_t i) { return !hdr[i].complete && !final; };
    auto take = [&](uint32_t i) {
        const RepHdr &h = rep[i];
        if (h.outcome == K4R_NONE || h.outcome == K4R_TRUNCATED) return;
        if (h.outcome == K4R_REPAIRED && h.data_off == 0xFFFFFFFFu) return;      /* no room in the pool: an overflow batch */
        wmb_repair_record r;
        memset(&r, 0, sizeof(r));
        r.sync_sample = hdr[i].sync_sample; r.end_sample = hdr[i].sync_sample + h.end_off;
        r.chain = hdr[i].chain; r.algo = hdr[i].algo; r.soft_t1 = (uint8_t)(h.had_line >> 1 & 1u);
        r.soft_s1 = (uint8_t)(h.had_line >> 2 & 1u);
        repaired_from(h, hdr[i].sync_sample, rep_mode(hdr[i].chain, dec[i]), pool, r.repair);
        fresh.push_back(r);
        if (h.outcome == K4R_REPAIRED && c->snip_mode) c->sn_ok[r.chain].insert(r.sync_sample);
        if (h.outcome == K4R_REPAIRED && c->telegrams) c->tg_rep.push_back(r);
    };
    /* the frames of a gather are in stream order: (chain, algo, ordinal) ascending */
    auto find = [&](int ch, int a, uint64_t ord) -> long {
        const FrameHdr *e = hdr + n;
        const FrameHdr *it = std::lower_bound(hdr, e, 0, [&](const FrameHdr &h, int) {
            if (h.chain != ch) return h.chain < ch;
            if (h.algo != a) return h.algo < a;
            return h.ordinal < ord;
        });
        return (it != e && it->chain == ch && it->algo == a && it->ordinal == ord && it->nbits) ? (long)(it - hdr) : -1;
    };
    for (int ch = 0; ch < WMB_N_CHAINS; ch++)
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            std::vector<uint64_t> &w = c->cb[ch].s[a].rep_wait;
            size_t keep = 0;
            for (uint64_t ord : w) {
                const long i = find(ch, a, ord);
                if (i < 0) continue;
                if (partial((uint32_t)i)) { w[keep++] = ord; continue; }
                take((uint32_t)i);
            }
            w.resize(keep);
        }
    for (size_t k : accepted) {
        const uint32_t i = idx[k];
        const FrameHdr &h = hdr[i];
        if (h.sync_sample < c->win_lo || h.sync_sample >= c->win_hi) continue;
        if (partial(i)) {
            /* a candidate whose list has not reached P yet (only an S1 abort can be booked so early) */
            if (rep[i].outcome == K4R_TRUNCATED) c->cb[h.chain].s[h.algo].rep_wait.push_back(h.ordinal);
            continue;
        }
        take(i);
    }
    std::sort(fresh.begin(), fresh.end(), [](const wmb_repair_record &x, const wmb_repair_record &y) {
        if (x.end_sample != y.end_sample) return x.end_sample < y.end_sample;
        const int px = x.chain * 2 + (x.algo == WMB_ALGO_T2A), py = y.chain * 2 + (y.algo == WMB_ALGO_T2A);
        if (px != py) return px < py;
        return x.sync_sample < y.sync_sample;
    });
    c->repairs.insert(c->repairs.end(), fresh.begin(), fresh.end());
}

/* candidates of one gathered batch, decoded by K4 (already in stream order); rep: K4R's verdicts when repair is on */
static int book_device_frames(wmb_ctx *c, const FrameHdr *hdr, const DecHdr *dec, const QualAcc *qual, const RepHdr *rep,
                              const uint8_t *pool, size_t n, bool final)
{
    /* frames without any bit (candidate at the very end of the stream) are not decoded at all */
    std::vector<uint32_t> idx;
    idx.reserve(n);
    for (size_t i = 0; i < n; i++) if (hdr[i].nbits) idx.push_back((uint32_t)i);
    std::vector<size_t> accepted;
    TRY(book_frames(c, idx.size(),
        [&](size_t k) {
            const FrameHdr &h = hdr[idx[k]];
            FrameMeta m;
            m.chain = h.chain; m.algo = h.algo; m.ordinal = h.ordinal; m.sync_sample = h.sync_sample;
            m.ofs_valid = 1; m.ofs_sum = h.ofs_sum; m.ofs_n = h.ofs_n;
            m.qual = qual ? qual + idx[k] : nullptr;
            m.partial = (uint8_t)((!h.complete && !final) ? 1 : 0);
            m.truncated = (uint8_t)((h.complete && !h.cut) ? 0 : 1);
            return m;
        },
        [&](size_t k) {
            const DecHdr &d = dec[idx[k]];
            DecLite l;
            l.status = d.status; l.consumed = d.consumed; l.end_sample = hdr[idx[k]].sync_sample + d.end_off; l.crc_ok = d.crc_ok;
            return l;
        },
        [&](size_t k, wmb_decoded &o) { decoded_from(dec[idx[k]], hdr[idx[k]].sync_sample, pool, o); },
        rep ? &accepted : nullptr));
    if (rep) book_repairs(c, hdr, dec, rep, pool, n, idx, accepted, final);
    return WMB_OK;
}

/* caller-made frames into the context's frame tables, and K4 on them; the datagram pool starts empty */
static int upload_and_decode(wmb_ctx *c, const wmb_frame *frames, size_t n)
{
    CUDA_TRY(cudaSetDevice(c->device));
    TRY(ctx_alloc(c));
    if (n > c->cand_cap) return set_err(WMB_E_INVAL, "too many frames");
    size_t words = 0;
    for (size_t i = 0; i < n; i++) {
        FrameHdr &h = c->hdr.h[i];
        memset(&h, 0, sizeof(h));
        h.ordinal = frames[i].ordinal; h.sync_sample = frames[i].sync_sample; h.nbits = frames[i].nbits;
        h.word_off = (uint32_t)words; h.chain = frames[i].chain; h.algo = frames[i].algo; h.complete = 1;
        if (words + h.nbits > c->frame_words_cap) return set_err(WMB_E_INVAL, "frames too large");
        memcpy(c->h_words + words, frames[i].bits, (size_t)h.nbits * 4);
        words += h.nbits;
    }
    CUDA_TRY(cudaMemcpyAsync(c->hdr.d, c->hdr.h, n * sizeof(FrameHdr), cudaMemcpyHostToDevice, c->cs));
    CUDA_TRY(cudaMemcpyAsync(c->d_words, c->h_words, words * 4, cudaMemcpyHostToDevice, c->cs));
    if (!c->inflight.empty()) return set_err(WMB_E_STATE, "unread results");
    CUDA_TRY(cudaMemsetAsync(GD_FIELD(c, pool_n), 0, 4, c->cs));
    K4Params q;
    memset(&q, 0, sizeof(q));
    q.hdr = c->hdr.d; q.n = (uint32_t)n; q.words = c->d_words; q.dec = c->dec.d;
    q.pool = c->pool.d; q.pool_cap = (uint32_t)c->pool.cap; q.pool_n = GD_FIELD(c, pool_n); q.errors = c->d_errors;
    return launch_k4(c, q);
}

/* Test hook (declared in wmb_framer.h, not part of the public ABI): run K4 on caller-made frames so
 * that the device framer can be compared with its host twin candidate by candidate. */
extern "C" int wmb_frame_decode_device(wmb_ctx *c, const wmb_frame *frames, size_t n, wmb_decoded *out)
{
    if (!c || !frames || !out) return set_err(WMB_E_INVAL, "null argument");
    TRY(upload_and_decode(c, frames, n));
    TRY(c->dec.fetch(0, 0, 0, (uint32_t)n, c->cs));
    TRY(c->pool.fetch(0, 0, 0, (uint32_t)std::min<size_t>(c->pool.cap, 1u << 24), c->cs));
    CUDA_TRY(cudaMemsetAsync(GD_FIELD(c, pool_n), 0, 4, c->cs));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    for (size_t i = 0; i < n; i++) decoded_from(c->dec.h[i], frames[i].sync_sample, c->pool.h, out[i]);
    return WMB_OK;
}

static int launch_k4r(wmb_ctx *c, const K4RParams &p)
{
#ifdef WMB_HOSTSIM
    static K4RSmem sm;                  /* the block's phases need real barriers: one simulated thread */
    hs_for(p.n, [&](uint32_t i) { k4r_repair(p, i, 0, 1, sm); });
#else
    k4r_repair_kernel<<<p.n ? p.n : 1, K4_THREADS, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
#endif
    c->st.kernel_launches += 1;
    return WMB_OK;
}

/* Test hook (wmbus_b200_framer.h): K4 and the erasure repair K4R on caller-made frames, to compare with the host twin
 * wmb_frame_repair() frame by frame. */
extern "C" int wmb_frame_repair_device(wmb_ctx *c, const wmb_frame *frames, size_t n, uint32_t e_max, wmb_repaired *out)
{
    if (!c || !frames || !out) return set_err(WMB_E_INVAL, "null argument");
    if (e_max > K4R_MAX_ERASURES) return set_err(WMB_E_INVAL, "e_max %u out of range 0..%d", e_max, K4R_MAX_ERASURES);
    memset(out, 0, n * sizeof(*out));
    if (e_max == 0 || n == 0) return WMB_OK;
    TRY(upload_and_decode(c, frames, n));
    RepHdr *d_rep = nullptr;
    if (cudaMalloc((void **)&d_rep, n * sizeof(RepHdr)) != cudaSuccess) return set_err(WMB_E_NOMEM, "cudaMalloc of the repair table failed");
    std::unique_ptr<RepHdr, cudaError_t (*)(void *)> guard(d_rep, cudaFree);
    K4RParams r;
    memset(&r, 0, sizeof(r));
    r.hdr = c->hdr.d; r.dec = c->dec.d; r.n = (uint32_t)n; r.words = c->d_words; r.rep = d_rep;
    r.pool = c->pool.d; r.pool_cap = (uint32_t)c->pool.cap; r.pool_n = GD_FIELD(c, pool_n); r.errors = c->d_errors;
    r.e_max = e_max;
    TRY(launch_k4r(c, r));
    std::vector<RepHdr> rep(n);
    CUDA_TRY(cudaMemcpyAsync(rep.data(), d_rep, n * sizeof(RepHdr), cudaMemcpyDeviceToHost, c->cs));
    TRY(c->pool.fetch(0, 0, 0, (uint32_t)std::min<size_t>(c->pool.cap, 1u << 24), c->cs));
    CUDA_TRY(cudaMemsetAsync(GD_FIELD(c, pool_n), 0, 4, c->cs));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    for (size_t i = 0; i < n; i++) {
        const RepHdr &h = rep[i];
        if (h.outcome == K4R_REPAIRED && h.data_off == 0xFFFFFFFFu)
            return set_err(WMB_E_OVERFLOW, "datagram pool full: hand in fewer frames at once");
        repaired_from(h, frames[i].sync_sample, frames[i].chain == WMB_CHAIN_T1C1 ? 0 : 2, c->pool.h, out[i]);
    }
    return WMB_OK;
}

static int launch_k4s(wmb_ctx *c, const K4SParams &p)
{
#ifdef WMB_HOSTSIM
    static K4SSmem sm;                  /* the block's phases need real barriers: one simulated thread */
    if (p.s1_max) hs_for(p.n, [&](uint32_t i) { k4s_repair<true>(p, i, 0, 1, sm); });
    else hs_for(p.n, [&](uint32_t i) { k4s_repair<false>(p, i, 0, 1, sm); });
#else
    if (p.s1_max) k4s_s1_repair_kernel<<<p.n ? p.n : 1, K4_THREADS, 0, c->cs>>>(p);
    else k4s_repair_kernel<<<p.n ? p.n : 1, K4_THREADS, 0, c->cs>>>(p);
    CUDA_TRY(cudaGetLastError());
#endif
    c->st.kernel_launches += 1;
    return WMB_OK;
}

/* K4, the erasure repair K4R and the soft repair K4S on caller-made frames, with one of K4S's limits (k_max: C1, s_max: T1,
 * s1_max: S1) set to k, named name in the messages; k = 0: wmb_frame_repair_device */
static int repair_soft_device(wmb_ctx *c, const wmb_frame *frames, const int16_t *const *softs, size_t n, uint32_t e_max,
                              uint32_t K4SParams::*limit, const char *name, uint32_t k, wmb_repaired *out)
{
    if (!c || !frames || !out || (!softs && n)) return set_err(WMB_E_INVAL, "null argument");
    if (k > WMB_SOFT_K_MAX) return set_err(WMB_E_INVAL, "%s %u out of range 0..%d", name, k, WMB_SOFT_K_MAX);
    if (k == 0) return wmb_frame_repair_device(c, frames, n, e_max, out);
    if (e_max > K4R_MAX_ERASURES) return set_err(WMB_E_INVAL, "e_max %u out of range 0..%d", e_max, K4R_MAX_ERASURES);
    memset(out, 0, n * sizeof(*out));
    if (n == 0) return WMB_OK;
    TRY(upload_and_decode(c, frames, n));
    std::vector<int16_t> hsoft;
    std::vector<uint8_t> hok(n);
    for (size_t i = 0; i < n; i++) {
        hok[i] = softs[i] ? 1 : 0;
        for (uint32_t j = 0; j < frames[i].nbits; j++) hsoft.push_back(softs[i] ? softs[i][j] : (int16_t)WMB_SOFT_NONE);
    }
    RepHdr *d_rep = nullptr;
    int16_t *d_soft = nullptr;
    uint8_t *d_ok = nullptr;
    if (cudaMalloc((void **)&d_rep, n * sizeof(RepHdr)) != cudaSuccess) return set_err(WMB_E_NOMEM, "cudaMalloc of the repair table failed");
    std::unique_ptr<RepHdr, cudaError_t (*)(void *)> guard(d_rep, cudaFree);
    if (cudaMalloc((void **)&d_soft, std::max<size_t>(hsoft.size(), 1) * 2) != cudaSuccess) return set_err(WMB_E_NOMEM, "cudaMalloc of the soft values failed");
    std::unique_ptr<int16_t, cudaError_t (*)(void *)> guard_s(d_soft, cudaFree);
    if (cudaMalloc((void **)&d_ok, n) != cudaSuccess) return set_err(WMB_E_NOMEM, "cudaMalloc of the soft flags failed");
    std::unique_ptr<uint8_t, cudaError_t (*)(void *)> guard_o(d_ok, cudaFree);
    CUDA_TRY(cudaMemcpyAsync(d_soft, hsoft.data(), hsoft.size() * 2, cudaMemcpyHostToDevice, c->cs));
    CUDA_TRY(cudaMemcpyAsync(d_ok, hok.data(), n, cudaMemcpyHostToDevice, c->cs));
    K4RParams r;
    memset(&r, 0, sizeof(r));
    r.hdr = c->hdr.d; r.dec = c->dec.d; r.n = (uint32_t)n; r.words = c->d_words; r.rep = d_rep;
    r.pool = c->pool.d; r.pool_cap = (uint32_t)c->pool.cap; r.pool_n = GD_FIELD(c, pool_n); r.errors = c->d_errors;
    r.e_max = e_max;
    if (e_max) TRY(launch_k4r(c, r));
    else CUDA_TRY(cudaMemsetAsync(d_rep, 0, n * sizeof(RepHdr), c->cs));      /* every record NONE, as K4R's off */
    K4SParams s;
    memset(&s, 0, sizeof(s));
    s.hdr = r.hdr; s.dec = r.dec; s.n = r.n; s.words = r.words; s.soft = d_soft; s.soft_ok = d_ok; s.rep = d_rep;
    s.pool = r.pool; s.pool_cap = r.pool_cap; s.pool_n = r.pool_n; s.errors = r.errors;
    s.*limit = k;
    TRY(launch_k4s(c, s));
    std::vector<RepHdr> rep(n);
    CUDA_TRY(cudaMemcpyAsync(rep.data(), d_rep, n * sizeof(RepHdr), cudaMemcpyDeviceToHost, c->cs));
    TRY(c->dec.fetch(0, 0, 0, (uint32_t)n, c->cs));                          /* (the mode of a repaired line) */
    TRY(c->pool.fetch(0, 0, 0, (uint32_t)std::min<size_t>(c->pool.cap, 1u << 24), c->cs));
    CUDA_TRY(cudaMemsetAsync(GD_FIELD(c, pool_n), 0, 4, c->cs));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    for (size_t i = 0; i < n; i++) {
        const RepHdr &h = rep[i];
        if (h.outcome == K4R_REPAIRED && h.data_off == 0xFFFFFFFFu)
            return set_err(WMB_E_OVERFLOW, "datagram pool full: hand in fewer frames at once");
        repaired_from(h, frames[i].sync_sample, rep_mode(frames[i].chain, c->dec.h[i]), c->pool.h, out[i]);
    }
    return WMB_OK;
}

/* Test hooks (wmbus_b200_framer.h): to compare with the host twins wmb_frame_repair_soft() / wmb_frame_repair_t1_soft()
 * frame by frame. */
extern "C" int wmb_frame_repair_soft_device(wmb_ctx *c, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                            uint32_t e_max, uint32_t k_max, wmb_repaired *out)
{
    return repair_soft_device(c, frames, softs, n, e_max, &K4SParams::k_max, "k_max", k_max, out);
}

extern "C" int wmb_frame_repair_t1_soft_device(wmb_ctx *c, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                               uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    return repair_soft_device(c, frames, softs, n, e_max, &K4SParams::s_max, "s_max", s_max, out);
}

extern "C" int wmb_frame_repair_s1_soft_device(wmb_ctx *c, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                               uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    return repair_soft_device(c, frames, softs, n, e_max, &K4SParams::s1_max, "s_max", s_max, out);
}

extern "C" int wmb_decode_frames(wmb_ctx *c, const wmb_frame *frames, size_t n)
{
    if (!c || (!frames && n)) return set_err(WMB_E_INVAL, "null argument");
    std::vector<const wmb_frame *> v(n);
    for (size_t i = 0; i < n; i++) v[i] = &frames[i];
    std::sort(v.begin(), v.end(), [](const wmb_frame *a, const wmb_frame *b) {
        if (a->chain != b->chain) return a->chain < b->chain;
        if (a->algo != b->algo) return a->algo < b->algo;
        return a->ordinal < b->ordinal;
    });
    for (const wmb_frame *f : v)
        if (f->chain >= WMB_N_CHAINS || f->algo >= WMB_N_ALGOS) return set_err(WMB_E_INVAL, "bad frame");
    /* frames handed in by the caller are decoded by the host twin of K4 (wmb_framer.c); the
     * per-frame decode is pure, so it is spread over a few host threads */
    std::vector<wmb_decoded> dec(n);
    {
        unsigned nt = n >= 256 ? std::min<unsigned>(8, std::max(1u, std::thread::hardware_concurrency())) : 1;
        auto work = [&](size_t lo, size_t hi) { for (size_t i = lo; i < hi; i++) wmb_frame_decode(v[i], &dec[i]); };
        if (nt <= 1) work(0, n);
        else {
            std::vector<std::thread> th;
            const size_t per = (n + nt - 1) / nt;
            for (unsigned t = 0; t < nt; t++) {
                const size_t lo = std::min(n, t * per), hi = std::min(n, lo + per);
                if (lo < hi) th.emplace_back(work, lo, hi);
            }
            for (auto &t : th) t.join();
        }
    }
    return book_frames(c, n,
        [&](size_t i) {
            FrameMeta m;
            m.chain = v[i]->chain; m.algo = v[i]->algo; m.ordinal = v[i]->ordinal; m.sync_sample = v[i]->sync_sample;
            m.partial = v[i]->reserved; m.truncated = v[i]->truncated;
            m.ofs_valid = 0; m.ofs_sum = 0; m.ofs_n = 0;                   /* a caller's frame carries no sum */
            m.qual = nullptr;
            return m;
        },
        [&](size_t i) {
            DecLite l;
            l.status = dec[i].status; l.consumed = dec[i].consumed; l.end_sample = dec[i].end_sample; l.crc_ok = dec[i].crc_ok;
            return l;
        },
        [&](size_t i, wmb_decoded &o) { o = dec[i]; });
}

/* deviation and eye SNR from the class sums (wmb_line_quality); returns valid */
static uint8_t qual_derive(const QualAcc &q, bool ok, double fir_gain, double *deviation_hz, double *eye_snr_db)
{
    *deviation_hz = NAN; *eye_snr_db = NAN;
    if (!ok || q.n_hi < 2 || q.n_lo < 2) return 0;
    const double nh = (double)q.n_hi, nl = (double)q.n_lo;
    const double mh = (double)q.s1_hi / nh, ml = (double)q.s1_lo / nl;
    const double var = ((double)q.s2_hi - nh * mh * mh + (double)q.s2_lo - nl * ml * ml) / (nh + nl - 2.0);
    if (!(var > 0.0)) return 0;
    const double half = (mh - ml) / 2.0;
    *deviation_hz = half / (double)WMB_OFS_SCALE * 400e3 / fir_gain;
    *eye_snr_db = 10.0 * log10(half * half / var);
    return 1;
}

extern "C" size_t wmb_take_lines_quality(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode,
                                         wmb_line_info *info, wmb_line_quality *qual, size_t rec_cap)
{
    size_t len = 0, taken = 0;
    if (n_lines) *n_lines = 0;
    if (!c || !buf) return 0;
    char ts[64];
    for (; taken < c->lines.size(); taken++) {
        if ((info || qual) && taken >= rec_cap) break;
        const QueuedLine &q = c->lines[taken];
        if (timestamp_mode == 1) snprintf(ts, sizeof(ts), "TS");
        else if (timestamp_mode == 2) snprintf(ts, sizeof(ts), "@%014llu.%d", (unsigned long long)q.end_sample, q.prio);
        else wmb_make_time_string(ts, sizeof(ts));
        const char *prefix = c->o.show_algorithm ? (q.algo == WMB_ALGO_RLA ? "rla;" : "t2a;") : "";
        char line[1024];
        const size_t l = wmb_format_line(&q.d, prefix, ts, line, sizeof(line));
        if (len + l + 1 > cap) break;
        memcpy(buf + len, line, l);
        len += l;
        if (info) {
            wmb_line_info &r = info[taken];
            memset(&r, 0, sizeof(r));
            r.sync_sample = q.sync_sample; r.end_sample = q.end_sample;
            r.chain = q.chain; r.algo = q.algo; r.crc_ok = q.d.crc_ok;
            /* -a: the cross-product discriminator is not a frequency */
            r.valid = (uint8_t)(q.ofs_valid && q.ofs_n > 0 && c->o.accurate_atan ? 1 : 0);
            r.n = q.ofs_n; r.sum = q.ofs_sum;
            r.carrier_hz = chain_carrier_hz(c, q.chain);
            r.offset_hz = r.valid ? (double)q.ofs_sum / (double)q.ofs_n / (double)WMB_OFS_SCALE * 400e3 / c->fir_gain[q.chain] : NAN;
        }
        if (qual) {
            wmb_line_quality &r = qual[taken];
            memset(&r, 0, sizeof(r));
            r.sync_sample = q.sync_sample; r.end_sample = q.end_sample;
            r.chain = q.chain; r.algo = q.algo; r.crc_ok = q.d.crc_ok;
            r.n_hi = q.qual.n_hi; r.n_lo = q.qual.n_lo; r.s1_hi = q.qual.s1_hi; r.s1_lo = q.qual.s1_lo;
            r.s2_hi = q.qual.s2_hi; r.s2_lo = q.qual.s2_lo;
            r.bits = q.d.consumed;
            /* -a: the cross-product discriminator is not a frequency; a caller's frame carries no sums */
            r.valid = qual_derive(q.qual, q.ofs_valid && c->o.accurate_atan, c->fir_gain[q.chain], &r.deviation_hz,
                                  &r.eye_snr_db);
            r.chip_rate_hz = (r.bits >= 2 && q.end_sample > q.sync_sample)
                ? 800e3 * (double)(r.bits - 1) / (double)(q.end_sample - q.sync_sample) : NAN;
        }
    }
    if (len < cap) buf[len] = 0;
    c->lines.erase(c->lines.begin(), c->lines.begin() + (long)taken);
    if (n_lines) *n_lines = taken;
    return len;
}

extern "C" size_t wmb_take_lines_info(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode,
                                      wmb_line_info *info, size_t info_cap)
{
    return wmb_take_lines_quality(c, buf, cap, n_lines, timestamp_mode, info, nullptr, info_cap);
}

extern "C" size_t wmb_take_lines(wmb_ctx *c, char *buf, size_t cap, size_t *n_lines, int timestamp_mode)
{
    return wmb_take_lines_info(c, buf, cap, n_lines, timestamp_mode, nullptr, 0);
}

extern "C" long wmb_process(wmb_ctx *c, const uint8_t *cu8, size_t nbytes, int flush,
                            char *out, size_t outcap, size_t *n_lines, int timestamp_mode)
{
    int rc = wmb_push(c, cu8, nbytes);
    if (rc) return rc;
    if (flush) {
        CUDA_TRY(cudaSetDevice(c->device));
        rc = flush_input(c);
        if (rc) return rc;
    }
    return (long)wmb_take_lines(c, out, outcap, n_lines, timestamp_mode);
}

extern "C" long wmb_process_device(wmb_ctx *c, const void *dev_cu8, size_t nbytes, int flush,
                                   char *out, size_t outcap, size_t *n_lines, int timestamp_mode)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (nbytes % 4096) return set_err(WMB_E_INVAL, "need a multiple of 4096 bytes");
    if (((uintptr_t)dev_cu8) & 15u) return set_err(WMB_E_INVAL, "device buffer must be 16-byte aligned");
    CUDA_TRY(cudaSetDevice(c->device));
    int rc = ctx_alloc(c);
    if (rc) return rc;
    tr("enter");
    rc = process_device_batches(c, (const uint8_t *)dev_cu8, nbytes, flush != 0);
    if (rc) return rc;
    tr("batches");
    if (flush) rc = flush_input(c);
    else rc = consume_all(c);
    if (rc) return rc;
    tr("flush");
    const long len = (long)wmb_take_lines(c, out, outcap, n_lines, timestamp_mode);
    tr("lines");
    tr_dump();
    return len;
}

/* Back to the state right after wmb_create (a new capture starts): filter memories, stream
 * position, pending candidates, queued lines.  Buffers stay allocated. */
extern "C" int wmb_reset(wmb_ctx *c)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    CUDA_TRY(cudaSetDevice(c->device));
    /* whatever was enqueued is abandoned: let it finish (a completed push has left the streams idle) */
    for (cudaStream_t st : { c->cs, c->xs, c->k1s, c->as[0], c->as[1], c->as2[0], c->as2[1], c->ts, c->s2, c->rs })
        if (st && cudaStreamQuery(st) != cudaSuccess) CUDA_TRY(cudaStreamSynchronize(st));
    c->iq_consumed = 0; c->m_consumed = 0; c->hist_m = 0; c->hist_iq = 0;
    c->remainder.clear(); c->lines.clear(); c->held.clear(); c->held_prev.clear(); c->repairs.clear();
    c->batch_no = 0; c->last_M = 0; c->prev_M = 0; c->last_hist = 0; c->last_set = 0; c->inflight.clear();
    c->chain_recorded[0] = c->chain_recorded[1] = false;
    c->stat_rerun_seen = 0; c->stat_fallback_seen = 0;
    c->bursts.clear(); c->burst_frontier = 0;
    c->sn_store.clear(); c->sn_queue.clear(); c->sn_ok[0].clear(); c->sn_ok[1].clear();
    c->sn_iq_end = 0; c->sn_g_first = 0; c->flushed = false;
    c->tg_info.clear(); c->tg_line.clear(); c->tg_rep.clear(); c->tg_ready.clear();
    c->spec_open = -1; c->spec_open_blocks = 0; c->spec_batch_rows.clear(); c->spec_enqueued = false;
    c->spec_rows.clear(); c->spec_sum.clear(); c->spec_peak.clear();
    for (int ch = 0; ch < WMB_N_CHAINS; ch++)
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            Stream &s = c->cb[ch].s[a];
            s.total = 0; s.total_prev = 0; s.busy_until = -1; s.rep_wait.clear();
        }
    if (c->allocated) {
        /* device state back to the start of a stream, in stream order on cs: one small kernel, no host copy, no wait;
         * the first batch's kernels on the other streams wait for it (ev_reset) */
        ResetParams r;
        memset(&r, 0, sizeof(r));
        for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
            if (!(c->chains & (1u << ch))) continue;
            r.ia_carry[ch] = c->cb[ch].ia_carry; r.rl_carry[ch] = c->cb[ch].rl_carry;
            for (int a = 0; a < WMB_N_ALGOS; a++) r.sd[ch * WMB_N_ALGOS + a] = c->cb[ch].s[a].sd;
        }
        r.gd = c->d_gd; r.errors = c->d_errors;
#ifdef WMB_HOSTSIM
        wmb_reset_device(r);
#else
        wmb_reset_kernel<<<1, 32, 0, c->cs>>>(r);
        CUDA_TRY(cudaGetLastError());
#endif
        if (c->burst_allocated)                  /* no run open */
            for (int ch = 0; ch < WMB_N_CHAINS; ch++)
                if (c->bb[ch].bd) CUDA_TRY(cudaMemsetAsync(c->bb[ch].bd, 0, sizeof(BurstDev), c->cs));
        if (c->d_snd) CUDA_TRY(cudaMemsetAsync(c->d_snd, 0, sizeof(SnipDev), c->cs));      /* no above granule yet */
        if (c->speak.cap) {                      /* no record open */
            CUDA_TRY(cudaMemsetAsync(c->d_ssum_ring, 0, c->speak.cap * sizeof(uint64_t), c->cs));
            CUDA_TRY(cudaMemsetAsync(c->d_speak_ring, 0, c->speak.cap * sizeof(uint32_t), c->cs));
        }
        CUDA_TRY(cudaEventRecord(c->ev_reset, c->cs));
        c->reset_pending = true;
    }
    return WMB_OK;
}

extern "C" int wmb_seek(wmb_ctx *c, uint64_t first_iq_sample)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (first_iq_sample % (2048ull * c->d)) return set_err(WMB_E_INVAL, "seek position must be a multiple of 2048 * decimation IQ samples");
    int rc = wmb_reset(c);
    if (rc) return rc;
    c->iq_consumed = first_iq_sample;
    c->m_consumed = first_iq_sample / c->d;
    c->sn_iq_end = first_iq_sample; c->sn_g_first = first_iq_sample / (2048ull * c->d);
    return WMB_OK;
}

extern "C" int wmb_set_receiver(wmb_ctx *c, int chain, uint32_t clock_lock, uint32_t access_code_errors)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (chain != WMB_CHAIN_T1C1 && chain != WMB_CHAIN_S1) return set_err(WMB_E_INVAL, "chain %d: 0 (T1/C1) or 1 (S1)", chain);
    if (clock_lock < 1 || clock_lock > WMB_LOCK_MAX)
        return set_err(WMB_E_INVAL, "clock lock %u out of range 1..%u", clock_lock, (unsigned)WMB_LOCK_MAX);
    const uint32_t emax = chain == WMB_CHAIN_T1C1 ? ChainT1C1::AC_ERR_MAX : ChainS1::AC_ERR_MAX;
    if (access_code_errors > emax)
        return set_err(WMB_E_INVAL, "access-code errors %u out of range 0..%u for the %s chain", access_code_errors, emax,
                       chain == WMB_CHAIN_T1C1 ? "T1/C1" : "S1");
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "wmb_set_receiver after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)");
    c->lock[chain] = clock_lock;
    c->ac_err[chain] = access_code_errors;
    return WMB_OK;
}

extern "C" int wmb_set_bursts(wmb_ctx *c, int chain, uint32_t level)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (chain != WMB_CHAIN_T1C1 && chain != WMB_CHAIN_S1) return set_err(WMB_E_INVAL, "chain %d: 0 (T1/C1) or 1 (S1)", chain);
    if (level > 255) return set_err(WMB_E_INVAL, "burst level %u out of range 0 (off) .. 255", level);
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "wmb_set_bursts after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)");
    c->burst_level[chain] = level;
    return WMB_OK;
}

extern "C" int wmb_take_bursts_quality(wmb_ctx *c, wmb_burst *out, wmb_burst_quality *qual, size_t cap, size_t *n)
{
    if (!c || !n || (!out && cap)) return set_err(WMB_E_INVAL, "null argument");
    /* per chain the queue is in start order (pieces of a chain are disjoint and close in order); across chains a
     * piece closed later may start earlier */
    std::stable_sort(c->bursts.begin(), c->bursts.end(), [](const QueuedBurst &a, const QueuedBurst &b) {
        return a.b.start_sample != b.b.start_sample ? a.b.start_sample < b.b.start_sample : a.b.chain < b.b.chain;
    });
    size_t k = 0;
    while (k < cap && k < c->bursts.size() && c->bursts[k].b.start_sample < c->burst_frontier) k++;
    for (size_t i = 0; i < k; i++) {
        const QueuedBurst &qb = c->bursts[i];
        out[i] = qb.b;
        if (!qual) continue;
        wmb_burst_quality &r = qual[i];
        memset(&r, 0, sizeof(r));
        r.start_sample = qb.b.start_sample; r.chain = qb.b.chain;
        r.n_hi = qb.q.n_hi; r.n_lo = qb.q.n_lo; r.s1_hi = qb.q.s1_hi; r.s1_lo = qb.q.s1_lo;
        r.s2_hi = qb.q.s2_hi; r.s2_lo = qb.q.s2_lo;
        r.valid = qual_derive(qb.q, c->o.accurate_atan != 0, c->fir_gain[qb.b.chain], &r.deviation_hz, &r.eye_snr_db);
    }
    c->bursts.erase(c->bursts.begin(), c->bursts.begin() + (long)k);
    *n = k;
    return WMB_OK;
}

extern "C" int wmb_take_bursts(wmb_ctx *c, wmb_burst *out, size_t cap, size_t *n)
{
    return wmb_take_bursts_quality(c, out, nullptr, cap, n);
}

extern "C" int wmb_set_line_quality(wmb_ctx *c, int on)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (on != 0 && on != 1) return set_err(WMB_E_INVAL, "line quality %d: 0 (off) or 1 (on)", on);
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "wmb_set_line_quality after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)");
    c->quality = on != 0;
    return WMB_OK;
}

/* What the repair and soft-value setters check alike: a context of the right kind (streaming for a repair setter, where
 * instead names the hook for polled frames; manual_frames for a soft-value setter, where instead names the streaming
 * setter), v in 0 (off) .. hi (what == null: the caller checked its value), and no sample pushed yet. */
static int repair_setter_check(wmb_ctx *c, const char *name, bool manual, const char *instead, const char *what, uint32_t v,
                               uint32_t hi)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (c->manual && !manual) return set_err(WMB_E_INVAL, "%s on a manual_frames context (repair the polled frames with %s)", name, instead);
    if (!c->manual && manual) return set_err(WMB_E_INVAL, "%s needs a manual_frames context (the streaming framer's %s)", name, instead);
    if (what && v > hi) return set_err(WMB_E_INVAL, "%s %u out of range 0 (off) .. %u", what, v, hi);
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "%s after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)", name);
    return WMB_OK;
}

extern "C" int wmb_set_repair(wmb_ctx *c, uint32_t e_max)
{
    TRY(repair_setter_check(c, "wmb_set_repair", false, "wmb_frame_repair_device", "e_max", e_max, K4R_MAX_ERASURES));
    c->repair_e = e_max;
    return WMB_OK;
}

extern "C" int wmb_set_soft_bits(wmb_ctx *c, int on)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (on != 0 && on != 1) return set_err(WMB_E_INVAL, "soft bits %d: 0 (off) or 1 (on)", on);
    TRY(repair_setter_check(c, "wmb_set_soft_bits", true, "soft repair: wmb_set_repair_soft", nullptr, 0, 0));
    c->soft = on != 0;
    return WMB_OK;
}

extern "C" int wmb_set_repair_soft(wmb_ctx *c, uint32_t k_max)
{
    TRY(repair_setter_check(c, "wmb_set_repair_soft", false, "wmb_frame_repair_soft_device", "k_max", k_max, WMB_SOFT_K_MAX));
    c->repair_k = k_max;
    return WMB_OK;
}

extern "C" int wmb_set_repair_t1_soft(wmb_ctx *c, uint32_t s_max)
{
    TRY(repair_setter_check(c, "wmb_set_repair_t1_soft", false, "wmb_frame_repair_t1_soft_device", "s_max", s_max, WMB_SOFT_K_MAX));
    c->repair_s = s_max;
    return WMB_OK;
}

extern "C" int wmb_set_soft_bits_s1(wmb_ctx *c, int on)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (on != 0 && on != 1) return set_err(WMB_E_INVAL, "S1 soft bits %d: 0 (off) or 1 (on)", on);
    TRY(repair_setter_check(c, "wmb_set_soft_bits_s1", true, "S1 soft repair: wmb_set_repair_s1_soft", nullptr, 0, 0));
    c->soft_s1 = on != 0;
    return WMB_OK;
}

extern "C" int wmb_set_repair_s1_soft(wmb_ctx *c, uint32_t s_max)
{
    TRY(repair_setter_check(c, "wmb_set_repair_s1_soft", false, "wmb_frame_repair_s1_soft_device", "s_max", s_max, WMB_SOFT_K_MAX));
    c->repair_s1 = s_max;
    return WMB_OK;
}

extern "C" int wmb_frame_soft(wmb_ctx *c, const wmb_frame *f, const int16_t **soft)
{
    if (!c || !f || !soft) return set_err(WMB_E_INVAL, "null argument");
    *soft = nullptr;
    for (const auto &h : c->held_prev)
        if (h.words.data() == f->bits) {
            if (!h.soft.empty()) *soft = h.soft.data();
            return WMB_OK;
        }
    return set_err(WMB_E_INVAL, "not a frame of the last wmb_poll");
}

extern "C" int wmb_take_repairs(wmb_ctx *c, wmb_repair_record *out, size_t cap, size_t *n)
{
    if (!c || !n || (!out && cap)) return set_err(WMB_E_INVAL, "null argument");
    const size_t k = std::min(cap, c->repairs.size());
    if (k) memcpy(out, c->repairs.data(), k * sizeof(wmb_repair_record));
    c->repairs.erase(c->repairs.begin(), c->repairs.begin() + (long)k);
    *n = k;
    return WMB_OK;
}

extern "C" int wmb_set_spectrum(wmb_ctx *c, uint32_t bins, uint32_t blocks_per_record)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (bins != 0) {
        if (bins != 256 && bins != 512 && bins != 1024 && bins != 2048)
            return set_err(WMB_E_INVAL, "spectrum bins %u: 256, 512, 1024 or 2048 (0: off)", bins);
        if (blocks_per_record < 1 || blocks_per_record > (1u << 20))
            return set_err(WMB_E_INVAL, "blocks per record %u out of range 1 .. 2^20", blocks_per_record);
        const uint64_t table = (uint64_t)spec_rows_for(c, bins, blocks_per_record) * bins;
        if (table > (1ull << 23))
            return set_err(WMB_E_INVAL, "spectrum table of %llu bins for %zu MiB batches (at most 2^23): raise blocks per record "
                           "or lower max_batch_mib", (unsigned long long)table, c->max_batch_bytes >> 20);
    }
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "wmb_set_spectrum after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)");
    c->spec_bins = bins;
    c->spec_B = bins ? blocks_per_record : 0;
    return WMB_OK;
}

extern "C" int wmb_take_spectrum(wmb_ctx *c, wmb_spectrum_row *rows, uint64_t *sum, float *peak, size_t cap, size_t *n)
{
    if (!c || !n || (cap && (!rows || !sum || !peak))) return set_err(WMB_E_INVAL, "null argument");
    const size_t k = std::min(cap, c->spec_rows.size());
    size_t bins = 0;
    for (size_t i = 0; i < k; i++) {
        rows[i] = c->spec_rows[i];
        memcpy(sum + bins, c->spec_sum.data() + bins, (size_t)rows[i].bins * sizeof(uint64_t));
        memcpy(peak + bins, c->spec_peak.data() + bins, (size_t)rows[i].bins * sizeof(float));
        bins += rows[i].bins;
    }
    c->spec_rows.erase(c->spec_rows.begin(), c->spec_rows.begin() + (long)k);
    c->spec_sum.erase(c->spec_sum.begin(), c->spec_sum.begin() + (long)bins);
    c->spec_peak.erase(c->spec_peak.begin(), c->spec_peak.begin() + (long)bins);
    *n = k;
    return WMB_OK;
}

extern "C" int wmb_debug_spectrum_tables(uint32_t bins, float *hann, float *tw)
{
    if (!hann || !tw || (bins != 256 && bins != 512 && bins != 1024 && bins != 2048)) return set_err(WMB_E_INVAL, "bad argument");
    spec_tables(bins, hann, tw);
    return WMB_OK;
}

extern "C" int wmb_set_line_window(wmb_ctx *c, uint64_t sync_lo, uint64_t sync_hi)
{
    if (!c || sync_lo > sync_hi) return set_err(WMB_E_INVAL, "bad window");
    c->win_lo = sync_lo; c->win_hi = sync_hi;
    return WMB_OK;
}

/* repair on: the candidate at ordinal ord of stream s is booked and waits for its repair (book_repairs) */
static bool rep_waiting(const wmb_ctx *c, const Stream &s, uint64_t ord)
{
    return c->repair_e && std::binary_search(s.rep_wait.begin(), s.rep_wait.end(), ord);
}

extern "C" long wmb_boundary_state(wmb_ctx *c, uint8_t *buf, size_t cap)
{
    if (!c || !buf) return set_err(WMB_E_INVAL, "null argument");
    if (!c->remainder.empty()) return set_err(WMB_E_STATE, "boundary state needs whole batch granules");
    CUDA_TRY(cudaSetDevice(c->device));
    int rc = ctx_alloc(c);
    if (rc) return rc;
    rc = consume_all(c);                                /* every enqueued batch is gathered and booked first */
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    GatherDev gd;
    CUDA_TRY(cudaMemcpy(&gd, c->d_gd, sizeof(gd), cudaMemcpyDeviceToHost));
    std::vector<uint8_t> out;
    auto put = [&](const void *p, size_t n) { const uint8_t *b = (const uint8_t *)p; out.insert(out.end(), b, b + n); };
    const uint64_t pos[2] = { c->iq_consumed, c->m_consumed };
    put(pos, sizeof(pos));
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!(c->chains & (1u << ch))) continue;
        ChainBuf &b = c->cb[ch];
        IirState ia;
        RlState rl;
        CUDA_TRY(cudaMemcpy(&ia, b.ia_carry, sizeof(ia), cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(&rl, b.rl_carry, sizeof(rl), cudaMemcpyDeviceToHost));
        if (!c->o.remove_dc) { ia.dc_x = 0.f; ia.dc_y = 0.f; }        /* unused without -o */
        if (!c->o.t2_enabled) memset(&ia, 0, sizeof(ia));
        if (!c->o.rla_enabled) memset(&rl, 0, sizeof(rl));
        ia.pad = 0;
        put(&ia, sizeof(ia));
        put(&rl, sizeof(rl));
        const uint32_t rx[2] = { c->lock[ch], c->ac_err[ch] };        /* contexts with other receiver settings never agree */
        put(rx, sizeof(rx));
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            if ((a == WMB_ALGO_RLA && !c->o.rla_enabled) || (a == WMB_ALGO_T2A && !c->o.t2_enabled)) continue;
            Stream &s = b.s[a];
            StreamDev sd;
            CUDA_TRY(cudaMemcpy(&sd, s.sd, sizeof(sd), cudaMemcpyDeviceToHost));
            const uint32_t sr = (a == WMB_ALGO_T2A) ? sd.t2_sr : 0u;
            put(&sr, 4);
            /* telegrams in flight: their bit events so far (sample, rssi, flags, bit are all in the word) */
            std::vector<uint64_t> pend(gd.n_pend[ch * WMB_N_ALGOS + a]);
            if (!pend.empty()) CUDA_TRY(cudaMemcpy(pend.data(), s.pend, pend.size() * 8, cudaMemcpyDeviceToHost));
            std::sort(pend.begin(), pend.end());
            const uint32_t np = (uint32_t)pend.size();
            put(&np, 4);
            for (uint64_t ord : pend) {
                if (ord >= sd.total) return set_err(WMB_E_STATE, "internal: pending candidate beyond the stream");
                const uint64_t n = sd.total - ord;
                if (n > WMB_MAXBITS + 64) return set_err(WMB_E_STATE, "internal: pending candidate older than a telegram");
                std::vector<uint64_t> ev((size_t)n);
                for (uint64_t i = 0; i < n;) {                         /* the ring wraps */
                    const uint64_t at = (ord + i) & (s.ring_cap - 1);
                    const uint64_t run = std::min<uint64_t>(n - i, s.ring_cap - at);
                    CUDA_TRY(cudaMemcpy(ev.data() + i, s.ring + at, (size_t)run * 8, cudaMemcpyDeviceToHost));
                    i += run;
                }
                /* a match inside a telegram that is already decoded will be ignored (busy decoder); bit 30: a candidate
                 * booked already that waits for its repair */
                const uint32_t n32 = (uint32_t)n | (((int64_t)ord <= s.busy_until) ? 0x80000000u : 0u)
                                   | (rep_waiting(c, s, ord) ? 0x40000000u : 0u);
                put(&n32, 4);
                put(ev.data(), ev.size() * 8);
            }
        }
    }
    if (c->repair_e) put(&c->repair_e, 4);             /* contexts that repair differently never agree */
    if (c->repair_k) put(&c->repair_k, 4);
    if (c->repair_s) { const uint8_t tag = 'T'; put(&tag, 1); put(&c->repair_s, 4); }   /* never reads as a k_max */
    if (c->repair_s1) { const uint8_t tag = 'S'; put(&tag, 1); put(&c->repair_s1, 4); }
    if (out.size() > cap) return set_err(WMB_E_INVAL, "buffer too small (%zu bytes needed)", out.size());
    memcpy(buf, out.data(), out.size());
    return (long)out.size();
}

/* the access-code matches (decimated samples) of the telegrams in flight, per chain; after consume_all */
static int pending_matches(wmb_ctx *c, std::vector<uint64_t> *match)
{
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    GatherDev gd;
    CUDA_TRY(cudaMemcpy(&gd, c->d_gd, sizeof(gd), cudaMemcpyDeviceToHost));
    std::vector<uint64_t> pend;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++) {
        if (!(c->chains & (1u << ch))) continue;
        for (int a = 0; a < WMB_N_ALGOS; a++) {
            if ((a == WMB_ALGO_RLA && !c->o.rla_enabled) || (a == WMB_ALGO_T2A && !c->o.t2_enabled)) continue;
            Stream &s = c->cb[ch].s[a];
            pend.resize(gd.n_pend[ch * WMB_N_ALGOS + a]);
            if (pend.empty()) continue;
            CUDA_TRY(cudaMemcpy(pend.data(), s.pend, pend.size() * 8, cudaMemcpyDeviceToHost));
            for (uint64_t ord : pend) {
                /* inside a telegram already decoded: will be ignored -- unless it is that telegram, waiting for its repair */
                if ((int64_t)ord <= s.busy_until && !rep_waiting(c, s, ord)) continue;
                uint64_t ev = 0;                                         /* the flagged bit's event: its sample is the match */
                CUDA_TRY(cudaMemcpy(&ev, s.ring + (ord & (s.ring_cap - 1)), 8, cudaMemcpyDeviceToHost));
                match[ch].push_back(c->m_consumed - ((c->m_consumed - EVG_M(ev)) & EVG_M_MASK));   /* 40 bits -> stream position */
            }
        }
    }
    return WMB_OK;
}

extern "C" long wmb_pending_before(wmb_ctx *c, uint64_t sync_hi)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    CUDA_TRY(cudaSetDevice(c->device));
    int rc = ctx_alloc(c);
    if (rc) return rc;
    rc = consume_all(c);                                /* every enqueued batch is gathered and booked first */
    if (rc) return rc;
    std::vector<uint64_t> match[WMB_N_CHAINS];
    rc = pending_matches(c, match);
    if (rc) return rc;
    long n_before = 0;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++)
        for (uint64_t m : match[ch]) if (m < sync_hi) n_before++;
    return n_before;
}

extern "C" int wmb_set_snippets(wmb_ctx *c, int mode)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (mode < 0 || mode > 2) return set_err(WMB_E_INVAL, "snippet mode %d: 0 (off), 1 (every burst) or 2 (undecoded bursts)", mode);
    if (c->batch_no != 0 || !c->remainder.empty())
        return set_err(WMB_E_STATE, "wmb_set_snippets after samples were pushed (call it before the first push or after wmb_reset / wmb_seek)");
    c->snip_mode = (uint32_t)mode;
    return WMB_OK;
}

/* a match of the chain's set in [lo, hi) */
static bool any_in(const std::set<uint64_t> &s, uint64_t lo, uint64_t hi)
{
    const auto it = s.lower_bound(lo);
    return it != s.end() && *it < hi;
}
static bool any_in(const std::vector<uint64_t> &v, uint64_t lo, uint64_t hi)
{
    for (uint64_t m : v) if (m >= lo && m < hi) return true;
    return false;
}

extern "C" int wmb_take_snippets(wmb_ctx *c, wmb_snippet *recs, size_t cap, uint8_t *bytes, size_t bytes_cap, size_t *n)
{
    if (!c || !n || (!recs && cap) || (!bytes && bytes_cap)) return set_err(WMB_E_INVAL, "null argument");
    *n = 0;
    if (!c->snip_mode || c->sn_queue.empty()) return WMB_OK;
    CUDA_TRY(cudaSetDevice(c->device));
    TRY(consume_all(c));
    /* per chain the queue is in start order; across chains a piece closed later may start earlier */
    std::stable_sort(c->sn_queue.begin(), c->sn_queue.end(), [](const wmb_snippet &a, const wmb_snippet &b) {
        return a.start_sample != b.start_sample ? a.start_sample < b.start_sample : a.chain < b.chain;
    });
    const uint64_t gi = 2048ull * c->d;
    const uint64_t g_whole = c->sn_iq_end / gi, g_end = (c->sn_iq_end + gi - 1) / gi;
    std::vector<uint64_t> pend[WMB_N_CHAINS];
    bool have_pend = c->flushed;                         /* nothing is in flight after the end of input */
    size_t k = 0, used = 0, i = 0;
    for (; i < c->sn_queue.size(); i++) {
        wmb_snippet q = c->sn_queue[i];
        if (q.start_sample >= c->burst_frontier) break;                  /* the burst report has not handed it out */
        if (!c->flushed && snip_hi(q.end_sample) > g_whole) break;       /* its last granules are still to come */
        if (!have_pend) { TRY(pending_matches(c, pend)); have_pend = true; }
        if (any_in(pend[q.chain], q.start_sample, q.end_sample)) break;  /* decoded or not is not known yet */
        q.decoded = any_in(c->sn_ok[q.chain], q.start_sample, q.end_sample) ? 1 : 0;
        if (q.decoded && c->snip_mode == 2) continue;
        const uint64_t lo = snip_lo(c, q.start_sample), hi = std::min(snip_hi(q.end_sample), g_end);
        uint64_t nb = 0;
        for (uint64_t g = lo; g < hi; g++) {
            const auto it = c->sn_store.find(g);
            if (it == c->sn_store.end() || it->second.lost) { q.lost = 1; break; }
            nb += it->second.bytes.size();
        }
        if (q.lost) nb = 0;
        if (k >= cap || used + nb > bytes_cap) break;
        q.start_iq = lo * gi; q.nbytes = nb;
        for (uint64_t g = lo; g < hi && !q.lost; g++) {
            const std::vector<uint8_t> &b = c->sn_store[g].bytes;
            memcpy(bytes + used, b.data(), b.size());
            used += b.size();
        }
        recs[k++] = q;
    }
    c->sn_queue.erase(c->sn_queue.begin(), c->sn_queue.begin() + (long)i);
    snip_prune(c);
    *n = k;
    return WMB_OK;
}

extern "C" int wmb_set_telegrams(wmb_ctx *c, int on)
{
    if (!c) return set_err(WMB_E_INVAL, "null argument");
    if (on != 0 && on != 1) return set_err(WMB_E_INVAL, "telegrams %d: 0 (off) or 1 (on)", on);
    if (c->manual) return set_err(WMB_E_INVAL, "wmb_set_telegrams on a manual_frames context (group its lines with wmb_group_telegrams)");
    TRY(repair_setter_check(c, "wmb_set_telegrams", false, nullptr, nullptr, 0, 0));
    c->telegrams = on != 0;
    return WMB_OK;
}

/* Telegrams: the groups of the kept candidates that are final go through wmb_group_telegrams into tg_ready.  A group
 * [lo, hi] of a chain is final when no match still to come can lie within W of it: a telegram in flight (its match is
 * known) outside [lo - W, hi + W], and a match not seen yet lies at or after the samples booked, m_consumed > hi + W.
 * Returns in *bound the sample before which no group still to come starts: the first match of the groups that are not
 * final, of the telegrams in flight, and m_consumed.  After consume_all. */
static int tlg_settle(wmb_ctx *c, uint64_t *bound)
{
    static const uint64_t W[WMB_N_CHAINS] = { WMB_TLG_W_T1C1, WMB_TLG_W_S1 };
    std::vector<uint64_t> pend[WMB_N_CHAINS];
    if (!c->flushed) TRY(pending_matches(c, pend));                   /* nothing is in flight after the end of input */
    const uint64_t seen = c->flushed ? ~0ull : c->m_consumed;
    *bound = seen;
    for (int ch = 0; ch < WMB_N_CHAINS; ch++)
        for (uint64_t p : pend[ch]) *bound = std::min(*bound, p);
    struct Cand { uint64_t sync; size_t i; uint8_t chain; };         /* i: line i, or repair record i - lines */
    const size_t nl = c->tg_info.size(), nr = c->tg_rep.size();
    std::vector<Cand> cand;
    cand.reserve(nl + nr);
    for (size_t i = 0; i < nl; i++) cand.push_back({ c->tg_info[i].sync_sample, i, c->tg_info[i].chain });
    for (size_t i = 0; i < nr; i++) cand.push_back({ c->tg_rep[i].sync_sample, nl + i, c->tg_rep[i].chain });
    std::sort(cand.begin(), cand.end(), [](const Cand &a, const Cand &b) {
        return a.chain != b.chain ? a.chain < b.chain : a.sync < b.sync;
    });
    std::vector<char> fin(nl + nr, 0);
    bool any = false;
    for (size_t g = 0, e; g < cand.size(); g = e) {
        const int ch = cand[g].chain;
        for (e = g + 1; e < cand.size() && cand[e].chain == ch && cand[e].sync - cand[e - 1].sync <= W[ch]; e++) {}
        const uint64_t lo = cand[g].sync, hi = cand[e - 1].sync;
        bool final = seen == ~0ull || hi + W[ch] < seen;
        for (uint64_t p : pend[ch]) if (p + W[ch] >= lo && p <= hi + W[ch]) final = false;
        if (!final) { *bound = std::min(*bound, lo); continue; }
        for (size_t k = g; k < e; k++) fin[cand[k].i] = 1;
        any = true;
    }
    if (!any) return WMB_OK;
    std::vector<wmb_line_info> info, keep_info;
    std::vector<wmb_decoded> line, keep_line;
    std::vector<wmb_repair_record> rep, keep_rep;
    size_t bytes = 0;
    for (size_t i = 0; i < nl; i++) {
        if (!fin[i]) { keep_info.push_back(c->tg_info[i]); keep_line.push_back(c->tg_line[i]); continue; }
        info.push_back(c->tg_info[i]); line.push_back(c->tg_line[i]);
        bytes += c->tg_line[i].len;
    }
    for (size_t i = 0; i < nr; i++) {
        if (!fin[nl + i]) { keep_rep.push_back(c->tg_rep[i]); continue; }
        rep.push_back(c->tg_rep[i]);
        bytes += c->tg_rep[i].repair.line.len;
    }
    std::vector<wmb_telegram> out(info.size() + rep.size());
    std::vector<uint8_t> data(bytes);
    size_t n = 0;
    if (wmb_group_telegrams(info.data(), line.data(), info.size(), rep.data(), rep.size(), out.data(), out.size(), data.data(),
                            data.size(), &n) != WMB_OK)
        return set_err(WMB_E_STATE, "internal: wmb_group_telegrams refused the context's candidates");
    size_t at = 0;
    for (size_t k = 0; k < n; k++) {
        c->tg_ready.push_back({ out[k], std::vector<uint8_t>(data.begin() + (long)at, data.begin() + (long)(at + out[k].len)) });
        at += out[k].len;
    }
    /* records of earlier groups may wait behind the bound; a group's records share (sync_sample, chain) */
    std::stable_sort(c->tg_ready.begin(), c->tg_ready.end(), [](const wmb_ctx::ReadyTelegram &a, const wmb_ctx::ReadyTelegram &b) {
        return a.t.sync_sample != b.t.sync_sample ? a.t.sync_sample < b.t.sync_sample : a.t.chain < b.t.chain;
    });
    c->tg_info.swap(keep_info); c->tg_line.swap(keep_line); c->tg_rep.swap(keep_rep);
    return WMB_OK;
}

extern "C" int wmb_take_telegrams(wmb_ctx *c, wmb_telegram *recs, size_t cap, uint8_t *data, size_t data_cap, size_t *n)
{
    if (!c || !n || (!recs && cap) || (!data && data_cap)) return set_err(WMB_E_INVAL, "null argument");
    *n = 0;
    if (!c->telegrams || (c->tg_info.empty() && c->tg_rep.empty() && c->tg_ready.empty())) return WMB_OK;
    CUDA_TRY(cudaSetDevice(c->device));
    TRY(consume_all(c));
    uint64_t bound = 0;
    TRY(tlg_settle(c, &bound));
    size_t k = 0, used = 0;
    for (; k < c->tg_ready.size() && k < cap; k++) {
        const wmb_ctx::ReadyTelegram &r = c->tg_ready[k];
        if (r.t.sync_sample >= bound || used + r.bytes.size() > data_cap) break;
        recs[k] = r.t;
        if (!r.bytes.empty()) memcpy(data + used, r.bytes.data(), r.bytes.size());
        used += r.bytes.size();
    }
    c->tg_ready.erase(c->tg_ready.begin(), c->tg_ready.begin() + (long)k);
    *n = k;
    return WMB_OK;
}

extern "C" int wmb_get_stats(wmb_ctx *c, wmb_stats *s)
{
    if (!c || !s) return set_err(WMB_E_INVAL, "null argument");
    *s = c->st;
    return WMB_OK;
}

extern "C" long wmb_debug_copy_stage(wmb_ctx *c, int chain, float *dphi, uint8_t *rssi, size_t cap)
{
    if (!c || chain < 0 || chain >= WMB_N_CHAINS || !c->allocated || !c->cb[chain].set[0].dphi)
        return set_err(WMB_E_INVAL, "stage not available");
    const SetBuf &sb = c->cb[chain].set[c->last_set];
    CUDA_TRY(cudaSetDevice(c->device));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    /* the last batch's outputs still sit at [W, W + last_M) until the next batch overwrites them */
    const size_t n = std::min<size_t>((size_t)c->last_M, cap);
    if (dphi) CUDA_TRY(cudaMemcpy(dphi, sb.dphi + c->W, n * 4, cudaMemcpyDeviceToHost));
    if (rssi) CUDA_TRY(cudaMemcpy(rssi, sb.rssi + c->W, n, cudaMemcpyDeviceToHost));
    return (long)n;
}

extern "C" long wmb_debug_copy_bits(wmb_ctx *c, int chain, int which, uint32_t *words, size_t cap_words)
{
    if (!c || chain < 0 || chain >= WMB_N_CHAINS || !words || !c->allocated || !c->cb[chain].set[0].dbits)
        return set_err(WMB_E_INVAL, "stage not available");
    const SetBuf &b = c->cb[chain].set[c->last_set];
    const uint32_t *src = which == 0 ? b.dbits : which == 1 ? b.sbits : which == 2 ? b.cbits : nullptr;
    if (!src) return set_err(WMB_E_INVAL, which == 2 ? "clock signs are kept only by a context created with opts.reserved[1] = 1" : "no such tap");
    CUDA_TRY(cudaSetDevice(c->device));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    const size_t n = std::min<size_t>(((size_t)c->last_M + 31) / 32, cap_words);
    CUDA_TRY(cudaMemcpy(words, src + c->W / 32, n * 4, cudaMemcpyDeviceToHost));
    return (long)n;
}

extern "C" long wmb_debug_copy_events(wmb_ctx *c, int chain, int algo, uint64_t *ev, size_t cap)
{
    if (!c || chain < 0 || chain >= WMB_N_CHAINS || algo < 0 || algo >= WMB_N_ALGOS || !ev || !c->allocated || !c->cb[chain].s[algo].ring)
        return set_err(WMB_E_INVAL, "stream not available");
    CUDA_TRY(cudaSetDevice(c->device));
    CUDA_TRY(cudaStreamSynchronize(c->cs));
    const Stream &s = c->cb[chain].s[algo];
    const uint64_t n = std::min<uint64_t>(s.total - s.total_prev, cap);
    if (s.total - s.total_prev > s.ring_cap) return set_err(WMB_E_OVERFLOW, "the batch wrote more events than the ring holds");
    for (uint64_t i = 0; i < n;) {                                   /* the ring wraps */
        const uint64_t at = (s.total_prev + i) & (s.ring_cap - 1);
        const uint64_t run = std::min<uint64_t>(n - i, s.ring_cap - at);
        CUDA_TRY(cudaMemcpy(ev + i, s.ring + at, (size_t)run * 8, cudaMemcpyDeviceToHost));
        i += run;
    }
    return (long)n;
}

/* Test hook: run the device's exact-arithmetic building blocks on caller-made operands (host arrays of n floats).
 * mode 0: bounded atan2f(y, x)   1: general atan2f(y, x)   2: bounded division y / x   3: bounded sqrt(y)
 *      4: discriminator of (y[i], x[i]) against (y[i-1], x[i-1]) taken as (I, Q) */
extern "C" int wmb_debug_arith(wmb_ctx *c, int mode, const float *y, const float *x, float *out, size_t n)
{
    if (!c || !y || !x || !out || mode < 0 || mode > 4) return set_err(WMB_E_INVAL, "bad argument");
#ifdef WMB_HOSTSIM
    WmbAtanTab tab;
    for (int i = 0; i < WMB_ATAN_TAB_ELEMS; i++) wmb_atan_tab_fill(&tab, i);
    for (size_t i = 0; i < n; i++)
        out[i] = mode == 0 ? wmb_atan2f_bounded(y[i], x[i], &tab) : mode == 1 ? wmb_atan2f(y[i], x[i])
               : mode == 2 ? wmb_fdiv_bounded(y[i], x[i]) : mode == 3 ? wmb_fsqrt_pos(y[i])
               : wmb_discriminator(y[i], x[i], y[i ? i - 1 : 0], x[i ? i - 1 : 0], &tab);
    return WMB_OK;
#else
    CUDA_TRY(cudaSetDevice(c->device));
    float *d = nullptr;
    CUDA_TRY(cudaMalloc(&d, 3 * n * sizeof(float) + 16));
    /* (everything on the context's stream: a plain cudaMemcpy from pageable memory may still be in flight on the
     * legacy stream when a kernel on a non-blocking stream starts) */
    cudaError_t e = cudaMemcpyAsync(d, y, n * 4, cudaMemcpyHostToDevice, c->cs);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + n, x, n * 4, cudaMemcpyHostToDevice, c->cs);
    if (e == cudaSuccess) { dbg_arith_kernel<<<1024, 256, 0, c->cs>>>(d, d + n, d + 2 * n, n, mode); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d + 2 * n, n * 4, cudaMemcpyDeviceToHost, c->cs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->cs);
    cudaFree(d);
    if (e != cudaSuccess) return set_err(WMB_E_CUDA, "wmb_debug_arith: %s", cudaGetErrorString(e));
    return WMB_OK;
#endif
}
