/*
 * rtl_wmbus_b200.c -- drop-in host program: same command line, stdin and stdout contract
 * as the reference's main() (rtl_wmbus.c:855-967 options/usage, :1217-1372 main loop),
 * with the per-sample work done by libwmbus_b200 on an H100.
 *
 *   rtl_sdr -f 868.95M -s 1600000 - 2>/dev/null | rtl_wmbus_b200
 *   cat capture.cu8 | rtl_wmbus_b200 -v
 *
 * stdin : interleaved unsigned 8-bit I/Q at decimation x 800 kS/s, consumed in whole
 *         4096-byte items (a trailing partial item is dropped, rtl_wmbus.c:1301-1308)
 * stdout: MODE;CRC_OK;3OUTOF6OK;TIMESTAMP;PACKET_RSSI;CURRENT_RSSI;LINK_LAYER_IDENT_NO;0xDATAGRAM
 * Extra environment knobs (not options, so the argv surface stays the reference's):
 *   WMBUS_B200_DEVICE=<n>      CUDA device (default 0)
 *   WMBUS_B200_BATCH_MIB=<n>   bytes gathered before a device pass (default 64)
 *   WMBUS_B200_CLOCK_LOCK=<t1c1>[,<s1>]           clock-lock threshold of the time2 algorithm, 1..16 (default 2,
 *                              the reference's opts_CLOCK_LOCK_THRESHOLD_*, rtl_wmbus.c:865-866)
 *   WMBUS_B200_ACCESS_CODE_ERRORS=<t1c1>[,<s1>]   access-code bit errors accepted, T1/C1 0..3, S1 0..6 (default 0,
 *                              ACCESS_CODE_*_ERRORS, rtl_wmbus.c:99, :103)
 *   One value sets both chains.  A malformed or out-of-range value is an error at start-up (wmb_set_receiver).
 *   WMBUS_B200_LINE_INFO=<path>  write one record per stdout line, in the same order and flushed with it:
 *                              ALGO;MODE;CRC_OK;LINK_LAYER_IDENT_NO;SYNC_SAMPLE;CARRIER_HZ;OFFSET_HZ (ALGO rla / t2a,
 *                              OFFSET_HZ the telegram's carrier offset from CARRIER_HZ, or nan; wmb_line_info).  A path
 *                              that cannot be opened is an error at start-up.  stdout does not change.
 *   WMBUS_B200_BURSTS=<path>   write one record per burst piece of either chain, decoded or not (wmb_take_bursts),
 *                              flushed after each hand-over: CHAIN;START_SAMPLE;END_SAMPLE;PEAK_RSSI;MEAN_RSSI;CARRIER_HZ;
 *                              OFFSET_HZ;FLAGS (CHAIN T1C1 / S1, OFFSET_HZ nan when not valid, FLAGS 1 continued, 2 cut,
 *                              4 at end of input).  A path that cannot be opened is an error at start-up.
 *   WMBUS_B200_BURST_LEVEL=<t1c1>[,<s1>]  the bursts' rssi level, 1..255 (0: that chain off; default 14).
 *   WMBUS_B200_SPECTRUM=<path> survey the whole captured band (wmb_set_spectrum) and write two lines per record, flushed
 *                              after each hand-over: mean;RECORD;START_IQ_SAMPLE;BLOCKS;HZ_LOW;HZ_STEP;dB_0;...;dB_{N-1}
 *                              with 10 log10(sum / blocks) per bin, then the same with peak and 10 log10(peak); HZ_LOW is
 *                              bin 0's frequency relative to the capture's centre.  tools/find_carriers.py reads the file.
 *   WMBUS_B200_SPECTRUM_BINS=<n>    bins N: 256, 512, 1024 (default) or 2048
 *   WMBUS_B200_SPECTRUM_BLOCKS=<n>  blocks of N IQ samples per record, 1 .. 2^20 (default 16384: 10.5 s at 1.6 MS/s)
 *   A path that cannot be opened or a bad value is an error at start-up.  stdout does not change.
 *   WMBUS_B200_LINE_QUALITY=<path>  write one record per stdout line, in the same order and flushed with it:
 *                              ALGO;MODE;CRC_OK;LINK_LAYER_IDENT_NO;SYNC_SAMPLE;DEVIATION_HZ;EYE_SNR_DB;CHIP_RATE_HZ
 *                              (wmb_line_quality; nan where not valid).
 *   WMBUS_B200_BURST_QUALITY=<path> (with WMBUS_B200_BURSTS) write one record per burst piece, in the burst file's
 *                              order: CHAIN;START_SAMPLE;DEVIATION_HZ;EYE_SNR_DB (wmb_burst_quality; nan where not valid).
 *   Either turns the quality report on (wmb_set_line_quality).  A path that cannot be opened is an error at start-up.
 *   WMBUS_B200_REPAIRED=<path> repair T1 and S1 telegrams that lost a few chips (wmb_set_repair) and write the line of
 *                              each repaired one, formatted as stdout's lines are (with the rla; / t2a; prefix under -v and
 *                              the wall-clock timestamp of the hand-over's stdout lines), flushed with stdout.
 *   WMBUS_B200_REPAIR_ERASURES=<n>  erasures repaired per CRC block, 1..3 (default 1: the lowest rate of wrong repairs,
 *                              DESIGN.md 8).  A path that cannot be opened, a bad value, or this variable without
 *                              WMBUS_B200_REPAIRED is an error at start-up.  stdout does not change.
 *   WMBUS_B200_REPAIR_SOFT_BITS=<k>  also repair C1 telegrams from the soft values of their bits, searching the k (1..6)
 *                              least reliable bits of each failing CRC block (wmb_set_repair_soft; DESIGN.md 8).  Unset:
 *                              C1 is not repaired.  A bad value, or this variable without WMBUS_B200_REPAIRED, is an
 *                              error at start-up.
 *   WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS=<s>  also repair T1 telegrams that erasure repair gives up on, from the soft values
 *                              of their chips: maximum-likelihood symbols and a search over the s (1..6) least confident
 *                              symbols of each failing CRC block (wmb_set_repair_t1_soft; DESIGN.md 8).  Unset: T1 is
 *                              repaired from hard decisions only.  A bad value, or this variable without
 *                              WMBUS_B200_REPAIRED, is an error at start-up.  stdout does not change.
 *   WMBUS_B200_REPAIR_S1_SOFT_BITS=<s>  also repair S1 telegrams that erasure repair gives up on, from the soft values
 *                              of their chips: maximum-likelihood bits and a search over the s (1..6) least reliable
 *                              Manchester pairs of each failing CRC block (wmb_set_repair_s1_soft; DESIGN.md 8).  Unset: S1
 *                              is repaired from hard decisions only.  A bad value, or this variable without
 *                              WMBUS_B200_REPAIRED, is an error at start-up.  stdout does not change.
 *   WMBUS_B200_SNIPPETS=<dir>  save the raw input around each burst piece (wmb_set_snippets, at the burst levels of
 *                              WMBUS_B200_BURST_LEVEL): after each hand-over one file <dir>/<START_IQ, 14 digits>_<T1C1|S1>.cu8
 *                              per snippet, and a line FILE;CHAIN;START_SAMPLE;END_SAMPLE;START_IQ;NBYTES;DECODED appended to
 *                              <dir>/snippets.txt (FILE "-" when the snippet was lost to a full device pool).  Pieces with
 *                              the same START_IQ share a file: the later one's snippet holds the earlier one's.  Piped back
 *                              with the same flags, a file prints the lines of its burst (but the TIMESTAMP column).
 *   WMBUS_B200_SNIPPET_MODE=undecoded|all   the pieces saved (default undecoded: those without a CRC-ok line).
 *   A directory that cannot be written, a bad mode, or a mode without WMBUS_B200_SNIPPETS is an error at start-up.
 *   stdout does not change.
 *   WMBUS_B200_TELEGRAMS=<path> write one record per transmission (wmb_set_telegrams: the lines of both bit syncs and,
 *                              with WMBUS_B200_REPAIRED, the repaired ones, grouped by their access-code matches), once
 *                              it is final, flushed after each hand-over:
 *                              MODE;DECODED;SOURCES;FAILED;SYNC_SAMPLE;MANUF;ID;VERSION;TYPE;CI;0xDATAGRAM
 *                              SOURCES the WMB_TLG_* bits (1 t2a line, 2 rla line, 4 t2a repair, 8 rla repair), ID %08X
 *                              (the LINK_LAYER_IDENT_NO of its lines), VERSION, TYPE and CI %02X.  A record with DECODED 0
 *                              has the chain (T1C1 or S1) as MODE and "-" for every field after SYNC_SAMPLE, and so has a
 *                              field the datagram is too short for.  A path that cannot be opened is an error at start-up.
 *                              stdout does not change.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <math.h>
#include <getopt.h>
#include <poll.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/time.h>
#include <time.h>
#include <unistd.h>

#include "wmbus_b200.h"
#include "wmbus_b200_framer.h"

static void print_usage(const char *program_name)
{
    /* same text as rtl_wmbus.c:869-884 */
    fprintf(stdout, "rtl_wmbus: %s\n\n", wmb_version_string());
    fprintf(stdout, "Usage %s:\n", program_name);
    fprintf(stdout, "\t-o remove DC offset\n");
    fprintf(stdout, "\t-a accelerate (use an inaccurate atan version)\n");
    fprintf(stdout, "\t-r 0 to disable run length algorithm\n");
    fprintf(stdout, "\t-t 0 to disable time2 algorithm\n");
    fprintf(stdout, "\t-d 2 set decimation rate to 2 (defaults to 2 if omitted)\n");
    fprintf(stdout, "\t-v show used algorithm in the output\n");
    fprintf(stdout, "\t-V show version\n");
    fprintf(stdout, "\t-s receive S1 and T1/C1 datagrams simultaneously. rtl_sdr _MUST_ be set to 868.625MHz (-f 868.625M)\n");
    fprintf(stdout, "\t-p [T,S] to disable processing T1/C1 or S1 mode\n");
    fprintf(stdout, "\t-f exit if flow of incoming data stops\n");
    fprintf(stdout, "\t-h print this help\n");
}

static void sig_alarm_handler(int signo)
{
    /* same message and exit status as rtl_wmbus.c:71-78.  The signal may be delivered to one of the CUDA runtime's
     * threads, where exit() would run the runtime's own exit handlers from inside itself: write() and _exit() instead
     * (stdout holds nothing: every line is flushed when it is printed). */
    static const char msg[] = "rtl_wmbus: exiting since incoming data stopped flowing!\n";
    (void)signo;
    if (write(STDERR_FILENO, msg, sizeof(msg) - 1) < 0) { /* nothing left to do about it */ }
    _exit(EXIT_FAILURE);
}

static double now_s(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* SIGALRM in `seconds` from now (0: cancel) */
static void set_alarm(double seconds)
{
    struct itimerval it;
    memset(&it, 0, sizeof(it));
    if (seconds > 0) {
        it.it_value.tv_sec = (time_t)seconds;
        it.it_value.tv_usec = (suseconds_t)((seconds - (double)(time_t)seconds) * 1e6);
        if (it.it_value.tv_sec == 0 && it.it_value.tv_usec == 0) it.it_value.tv_usec = 1;
    }
    setitimer(ITIMER_REAL, &it, NULL);
}

/* "<a>" or "<a>,<b>" of decimal numbers -> v[0], v[1] (one number: both); 0 if malformed */
static int parse_pair(const char *e, unsigned long v[2])
{
    char *end = NULL;
    if (e[0] < '0' || e[0] > '9') return 0;
    v[0] = v[1] = strtoul(e, &end, 10);
    if (*end == ',') {
        const char *f = end + 1;
        if (f[0] < '0' || f[0] > '9') return 0;
        v[1] = strtoul(f, &end, 10);
    }
    return *end == 0 && v[0] <= 0xFFFFFFFFul && v[1] <= 0xFFFFFFFFul;
}

#define STR_(x) #x
#define STR(x) STR_(x)
#define SOFT_K_MAX_STR STR(WMB_SOFT_K_MAX)

/* a WMBUS_B200_REPAIR_* variable: when set, it needs WMBUS_B200_REPAIRED and a decimal in 1 .. hi (expected says which)
 * goes to *v; returns 1 after printing why it does not */
static int repair_setting(const char *name, unsigned long hi, const char *expected, unsigned long *v)
{
    const char *e = getenv(name);
    if (!e) return 0;
    char *end = NULL;
    *v = strtoul(e, &end, 10);
    if (!getenv("WMBUS_B200_REPAIRED")) {
        fprintf(stderr, "rtl_wmbus_b200: %s needs WMBUS_B200_REPAIRED\n", name);
        return 1;
    }
    if (e[0] < '0' || e[0] > '9' || *end || *v < 1 || *v > hi) {
        fprintf(stderr, "rtl_wmbus_b200: %s=%s: expected %s\n", name, e, expected);
        return 1;
    }
    return 0;
}

/* WMBUS_B200_LINE_INFO / WMBUS_B200_LINE_QUALITY: one record per stdout line, in the same order */
static FILE *g_info_file = NULL, *g_qual_file = NULL;
#define INFO_CAP 4096
static wmb_line_info g_info[INFO_CAP];
static wmb_line_quality g_qual[INFO_CAP];

/* "%.<prec>f" of v, or nan */
static const char *fmt_or_nan(char *s, size_t cap, int valid, int prec, double v)
{
    if (valid && v == v) snprintf(s, cap, "%.*f", prec, v);
    else snprintf(s, cap, "nan");
    return s;
}

/* ALGO;MODE;CRC_OK;LINK_LAYER_IDENT_NO;SYNC_SAMPLE;CARRIER_HZ;OFFSET_HZ of each line of out[0..n) to the info file, and
 * ALGO;MODE;CRC_OK;LINK_LAYER_IDENT_NO;SYNC_SAMPLE;DEVIATION_HZ;EYE_SNR_DB;CHIP_RATE_HZ to the quality file */
static void write_info(const char *out, size_t n, size_t nl, int show_algorithm)
{
    const char *l = out;
    for (size_t i = 0; i < nl && l < out + n; i++) {
        const char *e = memchr(l, '\n', (size_t)(out + n - l));
        if (!e) e = out + n;
        /* fields of the line: [ALGO;]MODE;CRC_OK;3OUTOF6OK;TIMESTAMP;PACKET_RSSI;CURRENT_RSSI;LINK_LAYER_IDENT_NO;DATAGRAM */
        const char *f[9];
        int nf = 0;
        const char *p = l;
        if (show_algorithm) { p = memchr(p, ';', (size_t)(e - p)); p = p ? p + 1 : e; }
        while (nf < 9) {
            f[nf++] = p;
            const char *q = memchr(p, ';', (size_t)(e - p));
            if (!q) break;
            p = q + 1;
        }
        if (nf >= 8 && g_info_file) {
            const wmb_line_info *r = &g_info[i];
            char off[32];
            fprintf(g_info_file, "%s;%.*s;%u;%.*s;%llu;%.0f;%s\n", r->algo == WMB_ALGO_RLA ? "rla" : "t2a",
                    (int)(f[1] - f[0] - 1), f[0], (unsigned)r->crc_ok, (int)(f[7] - f[6] - 1), f[6],
                    (unsigned long long)r->sync_sample, r->carrier_hz, fmt_or_nan(off, sizeof(off), r->valid, 0, r->offset_hz));
        }
        if (nf >= 8 && g_qual_file) {
            const wmb_line_quality *r = &g_qual[i];
            char dev[32], snr[32], rate[32];
            fprintf(g_qual_file, "%s;%.*s;%u;%.*s;%llu;%s;%s;%s\n", r->algo == WMB_ALGO_RLA ? "rla" : "t2a",
                    (int)(f[1] - f[0] - 1), f[0], (unsigned)r->crc_ok, (int)(f[7] - f[6] - 1), f[6],
                    (unsigned long long)r->sync_sample, fmt_or_nan(dev, sizeof(dev), r->valid, 0, r->deviation_hz),
                    fmt_or_nan(snr, sizeof(snr), r->valid, 2, r->eye_snr_db),
                    fmt_or_nan(rate, sizeof(rate), 1, 1, r->chip_rate_hz));
        }
        l = e + 1;
    }
}

/* WMBUS_B200_BURSTS: one record per closed burst piece, CHAIN;START_SAMPLE;END_SAMPLE;PEAK_RSSI;MEAN_RSSI;CARRIER_HZ;
 * OFFSET_HZ;FLAGS.  The default level: the lowest at which the committed captures show no burst of noise alone, with
 * every CRC-ok line inside a burst (DESIGN.md 8) */
#define BURST_LEVEL_DEFAULT 14ul
static FILE *g_burst_file = NULL;
static const char *g_snip_dir /* WMBUS_B200_SNIPPETS */ = NULL;
static FILE *g_snip_index = NULL;
#define BURST_CAP 1024
static wmb_burst g_bursts[BURST_CAP];
/* WMBUS_B200_BURST_QUALITY: one record per burst piece, in the burst file's order: CHAIN;START_SAMPLE;DEVIATION_HZ;
 * EYE_SNR_DB */
static FILE *g_bqual_file = NULL;
static wmb_burst_quality g_bqual[BURST_CAP];

static void emit_bursts(wmb_ctx *ctx)
{
    if (!g_burst_file) {                                 /* on for the snippets alone: nobody reads the records */
        size_t n = 0;
        while (g_snip_dir && wmb_take_bursts(ctx, g_bursts, BURST_CAP, &n) == WMB_OK && n == BURST_CAP) {}
        return;
    }
    for (;;) {
        size_t n = 0;
        if (wmb_take_bursts_quality(ctx, g_bursts, g_bqual_file ? g_bqual : NULL, BURST_CAP, &n) != WMB_OK || !n) break;
        for (size_t i = 0; i < n; i++) {
            const wmb_burst *b = &g_bursts[i];
            char off[32];
            if (b->valid) snprintf(off, sizeof(off), "%.0f", b->offset_hz);
            else snprintf(off, sizeof(off), "nan");
            fprintf(g_burst_file, "%s;%llu;%llu;%u;%.1f;%.0f;%s;%u\n", b->chain == WMB_CHAIN_T1C1 ? "T1C1" : "S1",
                    (unsigned long long)b->start_sample, (unsigned long long)b->end_sample, (unsigned)b->peak,
                    (double)b->rssi_sum / (double)(b->end_sample - b->start_sample), b->carrier_hz, off, (unsigned)b->flags);
            if (g_bqual_file) {
                const wmb_burst_quality *q = &g_bqual[i];
                char dev[32], snr[32];
                fprintf(g_bqual_file, "%s;%llu;%s;%s\n", q->chain == WMB_CHAIN_T1C1 ? "T1C1" : "S1",
                        (unsigned long long)q->start_sample, fmt_or_nan(dev, sizeof(dev), q->valid, 0, q->deviation_hz),
                        fmt_or_nan(snr, sizeof(snr), q->valid, 2, q->eye_snr_db));
            }
        }
        if (n < BURST_CAP) break;
    }
    fflush(g_burst_file);
    if (g_bqual_file) fflush(g_bqual_file);
}

/* WMBUS_B200_SNIPPETS: one cu8 file per snippet and a line per snippet in the directory's index */
#define SNIP_CAP 256
#define SNIP_BYTES (32u << 20)                          /* > any one snippet: 101 granules of 4096 x 25 bytes */
static wmb_snippet g_snips[SNIP_CAP];
static uint8_t *g_snip_bytes = NULL;

static int emit_snippets(wmb_ctx *ctx)
{
    if (!g_snip_dir) return 0;
    for (;;) {
        size_t n = 0;
        if (wmb_take_snippets(ctx, g_snips, SNIP_CAP, g_snip_bytes, SNIP_BYTES, &n) != WMB_OK) {
            fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
            return -1;
        }
        if (!n) break;
        size_t at = 0;
        for (size_t i = 0; i < n; i++) {
            const wmb_snippet *q = &g_snips[i];
            const char *chain = q->chain == WMB_CHAIN_T1C1 ? "T1C1" : "S1";
            char name[64] = "-";
            if (!q->lost) {
                snprintf(name, sizeof(name), "%014llu_%s.cu8", (unsigned long long)q->start_iq, chain);
                char path[4096];
                snprintf(path, sizeof(path), "%s/%s", g_snip_dir, name);
                FILE *f = fopen(path, "wb");
                if (!f || fwrite(g_snip_bytes + at, 1, q->nbytes, f) != q->nbytes || fclose(f) != 0) {
                    fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SNIPPETS: %s: %s\n", path, strerror(errno));
                    return -1;
                }
                at += q->nbytes;
            }
            fprintf(g_snip_index, "%s;%s;%llu;%llu;%llu;%llu;%u\n", name, chain, (unsigned long long)q->start_sample,
                    (unsigned long long)q->end_sample, (unsigned long long)q->start_iq, (unsigned long long)q->nbytes,
                    q->decoded);
        }
    }
    return fflush(g_snip_index) == 0 ? 0 : -1;
}

/* WMBUS_B200_SPECTRUM: a mean line and a peak line per closed record of the band survey */
static FILE *g_spec_file = NULL;
#define SPEC_CAP 16
static wmb_spectrum_row g_spec_rows[SPEC_CAP];
static uint64_t g_spec_sum[SPEC_CAP * 2048];
static float g_spec_peak[SPEC_CAP * 2048];

static void emit_spectrum(wmb_ctx *ctx)
{
    if (!g_spec_file) return;
    for (;;) {
        size_t n = 0;
        if (wmb_take_spectrum(ctx, g_spec_rows, g_spec_sum, g_spec_peak, SPEC_CAP, &n) != WMB_OK || !n) break;
        for (size_t i = 0; i < n; i++) {
            const wmb_spectrum_row *r = &g_spec_rows[i];
            for (int pk = 0; pk < 2; pk++) {
                fprintf(g_spec_file, "%s;%llu;%llu;%u;%.2f;%.2f", pk ? "peak" : "mean", (unsigned long long)r->record,
                        (unsigned long long)r->start_iq, (unsigned)r->blocks, r->hz_low, r->hz_step);
                for (uint32_t k = 0; k < r->bins; k++) {
                    const double v = pk ? (double)g_spec_peak[i * r->bins + k]
                                        : (double)g_spec_sum[i * r->bins + k] / (double)r->blocks;
                    fprintf(g_spec_file, ";%.2f", 10.0 * log10(v));
                }
                fputc('\n', g_spec_file);
            }
        }
        if (n < SPEC_CAP) break;
    }
    fflush(g_spec_file);
}

/* WMBUS_B200_REPAIRED: the line of each REPAIRED record, with the timestamp of the hand-over's stdout lines */
static FILE *g_rep_file = NULL;
#define REP_CAP 256
static wmb_repair_record g_reps[REP_CAP];

static void emit_repairs(wmb_ctx *ctx, const char *ts, int show_algorithm)
{
    if (!g_rep_file) return;
    for (;;) {
        size_t n = 0;
        if (wmb_take_repairs(ctx, g_reps, REP_CAP, &n) != WMB_OK || !n) break;
        for (size_t i = 0; i < n; i++) {
            const wmb_repair_record *r = &g_reps[i];
            if (r->repair.outcome != WMB_REP_REPAIRED) continue;
            char line[1024];
            const char *prefix = show_algorithm ? (r->algo == WMB_ALGO_RLA ? "rla;" : "t2a;") : "";
            fwrite(line, 1, wmb_format_line(&r->repair.line, prefix, ts, line, sizeof(line)), g_rep_file);
        }
        if (n < REP_CAP) break;
    }
    fflush(g_rep_file);
}

/* WMBUS_B200_TELEGRAMS: one line per final telegram record */
static FILE *g_tlg_file = NULL;
#define TLG_CAP 256
static wmb_telegram g_tlgs[TLG_CAP];
static uint8_t g_tlg_bytes[TLG_CAP * 292];

static void put_field(uint8_t valid, uint8_t bit, const char *fmt, unsigned v)
{
    if (valid & bit) fprintf(g_tlg_file, fmt, v);
    else fputs(";-", g_tlg_file);
}

static int emit_telegrams(wmb_ctx *ctx)
{
    if (!g_tlg_file) return 0;
    for (;;) {
        size_t n = 0;
        if (wmb_take_telegrams(ctx, g_tlgs, TLG_CAP, g_tlg_bytes, sizeof(g_tlg_bytes), &n) != WMB_OK) {
            fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
            return -1;
        }
        if (!n) break;
        size_t at = 0;
        for (size_t i = 0; i < n; i++) {
            const wmb_telegram *t = &g_tlgs[i];
            const char *mode = t->decoded ? t->mode : t->chain == WMB_CHAIN_T1C1 ? "T1C1" : "S1";
            fprintf(g_tlg_file, "%s;%u;%u;%u;%llu", mode, t->decoded, t->sources, t->failed, (unsigned long long)t->sync_sample);
            if (t->valid & WMB_TLG_F_M) fprintf(g_tlg_file, ";%s", t->manuf);
            else fputs(";-", g_tlg_file);
            put_field(t->valid, WMB_TLG_F_ID, ";%08X", t->id);
            put_field(t->valid, WMB_TLG_F_VERSION, ";%02X", t->version);
            put_field(t->valid, WMB_TLG_F_TYPE, ";%02X", t->type);
            put_field(t->valid, WMB_TLG_F_CI, ";%02X", t->ci);
            if (t->len) {
                fputs(";0x", g_tlg_file);
                for (unsigned k = 0; k < t->len; k++) fprintf(g_tlg_file, "%02x", g_tlg_bytes[at + k]);
                fputc('\n', g_tlg_file);
            } else fputs(";-\n", g_tlg_file);
            at += t->len;
        }
    }
    return fflush(g_tlg_file) == 0 ? 0 : -1;
}

static int emit_lines(wmb_ctx *ctx, char *out, size_t outcap, int show_algorithm)
{
    if (emit_snippets(ctx)) return -1;
    emit_bursts(ctx);
    emit_spectrum(ctx);
    /* the repaired lines carry the hand-over's wall-clock time, taken as its stdout lines are formatted */
    char ts[64];
    wmb_make_time_string(ts, sizeof(ts));
    for (;;) {
        size_t nl = 0;
        const size_t n = g_info_file || g_qual_file
            ? wmb_take_lines_quality(ctx, out, outcap, &nl, 0, g_info_file ? g_info : NULL, g_qual_file ? g_qual : NULL, INFO_CAP)
            : wmb_take_lines(ctx, out, outcap, &nl, 0);
        if (!nl) {
            emit_repairs(ctx, ts, show_algorithm);
            return emit_telegrams(ctx);
        }
        fwrite(out, 1, n, stdout);
        fflush(stdout);                                 /* t1_c1_packet_decoder.h:698-699 */
        if (g_info_file || g_qual_file) {
            write_info(out, n, nl, show_algorithm);
            if (g_info_file) fflush(g_info_file);
            if (g_qual_file) fflush(g_qual_file);
        }
    }
}

int main(int argc, char *argv[])
{
    wmb_opts o;
    int check_flow = 0, option;
    wmb_default_opts(&o);

    if (argc == 1 && isatty(0)) {                       /* rtl_wmbus.c:1223-1228 */
        print_usage(argv[0]);
        exit(0);
    }

    while ((option = getopt(argc, argv, "ofad:p:r:vVst:")) != -1) {   /* rtl_wmbus.c:896 */
        switch (option) {
        case 'o': o.remove_dc = 1; break;
        case 'f': check_flow = 1; break;
        case 'a': o.accurate_atan = 0; break;
        case 'p':
            if (strcmp(optarg, "T") == 0 || strcmp(optarg, "t") == 0) o.t1c1_enabled = 0;
            else if (strcmp(optarg, "S") == 0 || strcmp(optarg, "s") == 0) o.s1_enabled = 0;
            else { print_usage(argv[0]); exit(EXIT_FAILURE); }
            break;
        case 'r':
            if (strcmp(optarg, "0") == 0) o.rla_enabled = 0;
            else { print_usage(argv[0]); exit(EXIT_FAILURE); }
            break;
        case 't':
            if (strcmp(optarg, "0") == 0) o.t2_enabled = 0;
            else { print_usage(argv[0]); exit(EXIT_FAILURE); }
            break;
        case 'd': o.decimation = (uint32_t)strtoul(optarg, NULL, 10); break;
        case 's': o.simultaneous = 1; break;
        case 'v': o.show_algorithm = 1; break;
        case 'V':
            fprintf(stdout, "rtl_wmbus: %s\n", wmb_version_string());
            fprintf(stdout, "libwmbus_b200 ABI %d\n", wmb_abi_version());
            exit(EXIT_SUCCESS);
        default:
            print_usage(argv[0]);
            exit(EXIT_FAILURE);
        }
    }

    if (check_flow) {                                   /* rtl_wmbus.c:1238-1246 */
        struct sigaction new_alarm;
        new_alarm.sa_handler = sig_alarm_handler;
        sigemptyset(&new_alarm.sa_mask);
        new_alarm.sa_flags = 0;
        fprintf(stderr, "rtl_wmbus: monitoring flow\n");
        sigaction(SIGALRM, &new_alarm, NULL);
    }

    const char *e;
    const int device = (e = getenv("WMBUS_B200_DEVICE")) ? atoi(e) : 0;
    unsigned long batch_mib = 64;
    if ((e = getenv("WMBUS_B200_BATCH_MIB")) != NULL) {
        char *end = NULL;
        const unsigned long v = strtoul(e, &end, 10);
        if (end != e && *end == 0 && e[0] != '-') batch_mib = v;
    }
    if (batch_mib < 1) batch_mib = 1;
    if (batch_mib > 1024) batch_mib = 1024;
    const size_t batch = (size_t)batch_mib * 1048576u;
    o.max_batch_mib = (uint32_t)batch_mib;

    unsigned long lock[2] = { 2, 2 }, errors[2] = { 0, 0 };
    if ((e = getenv("WMBUS_B200_CLOCK_LOCK")) != NULL && !parse_pair(e, lock)) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_CLOCK_LOCK=%s: expected <t1c1>[,<s1>]\n", e);
        return EXIT_FAILURE;
    }
    if ((e = getenv("WMBUS_B200_ACCESS_CODE_ERRORS")) != NULL && !parse_pair(e, errors)) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_ACCESS_CODE_ERRORS=%s: expected <t1c1>[,<s1>]\n", e);
        return EXIT_FAILURE;
    }

    unsigned long burst_level[2] = { BURST_LEVEL_DEFAULT, BURST_LEVEL_DEFAULT };
    if ((e = getenv("WMBUS_B200_BURST_LEVEL")) != NULL && (!parse_pair(e, burst_level) || burst_level[0] > 255 || burst_level[1] > 255)) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURST_LEVEL=%s: expected <t1c1>[,<s1>], 0 (off) .. 255\n", e);
        return EXIT_FAILURE;
    }
    if ((e = getenv("WMBUS_B200_BURSTS")) != NULL && (g_burst_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURSTS=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }

    unsigned long spec_bins = 1024, spec_blocks = 16384;
    if ((e = getenv("WMBUS_B200_SPECTRUM_BINS")) != NULL) {
        char *end = NULL;
        spec_bins = strtoul(e, &end, 10);
        if (e[0] < '0' || e[0] > '9' || *end || (spec_bins != 256 && spec_bins != 512 && spec_bins != 1024 && spec_bins != 2048)) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SPECTRUM_BINS=%s: expected 256, 512, 1024 or 2048\n", e);
            return EXIT_FAILURE;
        }
    }
    if ((e = getenv("WMBUS_B200_SPECTRUM_BLOCKS")) != NULL) {
        char *end = NULL;
        spec_blocks = strtoul(e, &end, 10);
        if (e[0] < '0' || e[0] > '9' || *end || spec_blocks < 1 || spec_blocks > (1ul << 20)) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SPECTRUM_BLOCKS=%s: expected 1 .. 1048576\n", e);
            return EXIT_FAILURE;
        }
    }
    if ((e = getenv("WMBUS_B200_SPECTRUM")) != NULL && (g_spec_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SPECTRUM=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }

    if ((e = getenv("WMBUS_B200_LINE_INFO")) != NULL && (g_info_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_LINE_INFO=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }
    if ((e = getenv("WMBUS_B200_LINE_QUALITY")) != NULL && (g_qual_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_LINE_QUALITY=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }
    if ((e = getenv("WMBUS_B200_BURST_QUALITY")) != NULL) {
        if (!g_burst_file) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURST_QUALITY needs WMBUS_B200_BURSTS\n");
            return EXIT_FAILURE;
        }
        if ((g_bqual_file = fopen(e, "w")) == NULL) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURST_QUALITY=%s: %s\n", e, strerror(errno));
            return EXIT_FAILURE;
        }
    }

    int snip_mode = 0;
    if ((e = getenv("WMBUS_B200_SNIPPET_MODE")) != NULL) {
        if (strcmp(e, "undecoded") == 0) snip_mode = 2;
        else if (strcmp(e, "all") == 0) snip_mode = 1;
        else {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SNIPPET_MODE=%s: expected undecoded or all\n", e);
            return EXIT_FAILURE;
        }
        if (!getenv("WMBUS_B200_SNIPPETS")) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SNIPPET_MODE needs WMBUS_B200_SNIPPETS\n");
            return EXIT_FAILURE;
        }
    }
    if ((g_snip_dir = getenv("WMBUS_B200_SNIPPETS")) != NULL) {
        char path[4096];
        snprintf(path, sizeof(path), "%s/snippets.txt", g_snip_dir);
        if ((g_snip_index = fopen(path, "a")) == NULL) {
            fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SNIPPETS=%s: %s\n", g_snip_dir, strerror(errno));
            return EXIT_FAILURE;
        }
        if (!snip_mode) snip_mode = 2;
        if ((g_snip_bytes = malloc(SNIP_BYTES)) == NULL) {
            fprintf(stderr, "rtl_wmbus_b200: out of memory\n");
            return EXIT_FAILURE;
        }
    }

    unsigned long repair_e = 1, repair_k = 0, repair_s = 0, repair_s1 = 0;
    if (repair_setting("WMBUS_B200_REPAIR_ERASURES", 3, "1, 2 or 3", &repair_e) ||
        repair_setting("WMBUS_B200_REPAIR_SOFT_BITS", WMB_SOFT_K_MAX, "1 .. " SOFT_K_MAX_STR, &repair_k) ||
        repair_setting("WMBUS_B200_REPAIR_T1_SOFT_SYMBOLS", WMB_SOFT_K_MAX, "1 .. " SOFT_K_MAX_STR, &repair_s) ||
        repair_setting("WMBUS_B200_REPAIR_S1_SOFT_BITS", WMB_SOFT_K_MAX, "1 .. " SOFT_K_MAX_STR, &repair_s1))
        return EXIT_FAILURE;
    if ((e = getenv("WMBUS_B200_REPAIRED")) != NULL && (g_rep_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_REPAIRED=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }

    if ((e = getenv("WMBUS_B200_TELEGRAMS")) != NULL && (g_tlg_file = fopen(e, "w")) == NULL) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_TELEGRAMS=%s: %s\n", e, strerror(errno));
        return EXIT_FAILURE;
    }

    wmb_ctx *ctx = NULL;
    if (wmb_create(&o, device, &ctx) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    for (int ch = 0; ch < 2; ch++)
        if (wmb_set_receiver(ctx, ch, (uint32_t)lock[ch], (uint32_t)errors[ch]) != WMB_OK) {
            fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
            return EXIT_FAILURE;
        }
    if (g_burst_file || g_snip_dir)
        for (int ch = 0; ch < 2; ch++)
            if (wmb_set_bursts(ctx, ch, (uint32_t)burst_level[ch]) != WMB_OK) {
                fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
                return EXIT_FAILURE;
            }
    if ((g_qual_file || g_bqual_file) && wmb_set_line_quality(ctx, 1) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    if (g_rep_file && (wmb_set_repair(ctx, (uint32_t)repair_e) != WMB_OK || wmb_set_repair_soft(ctx, (uint32_t)repair_k) != WMB_OK ||
                       wmb_set_repair_t1_soft(ctx, (uint32_t)repair_s) != WMB_OK ||
                       wmb_set_repair_s1_soft(ctx, (uint32_t)repair_s1) != WMB_OK)) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    if (g_tlg_file && wmb_set_telegrams(ctx, 1) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    if (g_snip_dir && wmb_set_snippets(ctx, snip_mode) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    if (g_spec_file && wmb_set_spectrum(ctx, (uint32_t)spec_bins, (uint32_t)spec_blocks) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SPECTRUM: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }
    uint8_t *buf = wmb_host_alloc(batch);
    const size_t outcap = 1u << 20;
    char *out = malloc(outcap);
    if (!buf || !out) {
        fprintf(stderr, "rtl_wmbus_b200: out of memory\n");
        return EXIT_FAILURE;
    }

    /* device buffers are allocated at the first push: do it now, not when the first samples are waiting */
    if (wmb_push(ctx, buf, 0) != WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
        return EXIT_FAILURE;
    }

    size_t fill = 0;
    /* -f: the reference arms a 2 s alarm around each fread() of one 4096-byte item (rtl_wmbus.c:1300-1302), i.e. it
     * gives up when a whole item does not arrive within 2 s -- a trickle of bytes does not keep it alive.  Here the
     * reads are whatever the pipe holds, so the alarm stays armed until 4096 new bytes have come in since it was set;
     * it is not running while the device works on a hand-over. */
    size_t since_arm = 0;
    int armed = 0;
    double deadline = 0;
    double last_push = now_s();
    int rc = WMB_OK, eof = 0;
    while (!eof) {
        /* wait for input; on a live stream hand over what has arrived every 100 ms so
         * that telegrams are printed promptly */
        struct pollfd pfd = { 0, POLLIN, 0 };
        if (check_flow && !armed) { deadline = now_s() + 2.0; set_alarm(2.0); armed = 1; since_arm = 0; }      /* START_ALARM */
        const int pr = poll(&pfd, 1, fill ? 100 : -1);
        ssize_t n = 0;
        if (pr > 0) {
            n = read(0, buf + fill, batch - fill);
            if (n < 0 && errno == EINTR) n = 0;
            else if (n <= 0) eof = 1;
            else { fill += (size_t)n; since_arm += (size_t)n; }
        } else if (pr < 0 && errno != EINTR) {
            eof = 1;
        }
        if (check_flow && armed && (since_arm >= 4096 || eof)) { set_alarm(0); armed = 0; }     /* STOP_ALARM: an item is in */
        const double t = now_s();
        if (fill == batch || eof || (fill && (pr == 0 || t - last_push > 0.1))) {
            if (check_flow && armed) {                  /* the watchdog times the input, not the device */
                set_alarm(0);
                const double t_in = now_s();
                rc = wmb_push(ctx, buf, fill);
                if (rc == WMB_OK && emit_lines(ctx, out, outcap, o.show_algorithm)) rc = WMB_E_STATE;
                deadline += now_s() - t_in;             /* the item's two seconds do not run during the hand-over */
                const double left = deadline - now_s();
                set_alarm(left > 1e-3 ? left : 1e-3);
            } else {
                rc = wmb_push(ctx, buf, fill);
                if (rc == WMB_OK && emit_lines(ctx, out, outcap, o.show_algorithm)) rc = WMB_E_STATE;
            }
            if (rc != WMB_OK) break;
            fill = 0;
            last_push = t;
        }
    }
    if (check_flow) set_alarm(0);
    if (rc == WMB_OK) {
        size_t nframes = 0;
        rc = wmb_poll(ctx, NULL, 0, &nframes, 1);       /* EOF: flush */
        if (rc == WMB_OK && emit_lines(ctx, out, outcap, o.show_algorithm)) rc = WMB_E_STATE;
    }
    if (rc != WMB_OK) fprintf(stderr, "rtl_wmbus_b200: %s\n", wmb_last_error());
    free(out);
    wmb_host_free(buf);
    wmb_destroy(ctx);
    if (g_spec_file && fclose(g_spec_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SPECTRUM: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_burst_file && fclose(g_burst_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURSTS: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_info_file && fclose(g_info_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_LINE_INFO: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_qual_file && fclose(g_qual_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_LINE_QUALITY: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_bqual_file && fclose(g_bqual_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_BURST_QUALITY: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_snip_index && fclose(g_snip_index) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_SNIPPETS: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    free(g_snip_bytes);
    if (g_tlg_file && fclose(g_tlg_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_TELEGRAMS: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    if (g_rep_file && fclose(g_rep_file) != 0 && rc == WMB_OK) {
        fprintf(stderr, "rtl_wmbus_b200: WMBUS_B200_REPAIRED: %s\n", strerror(errno));
        return EXIT_FAILURE;
    }
    return rc == WMB_OK ? EXIT_SUCCESS : EXIT_FAILURE;
}
