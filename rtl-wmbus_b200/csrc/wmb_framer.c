/*
 * wmb_framer.c -- host-side T1 / C1 (frame A, B) / S1 framers of libwmbus_b200.
 *
 * The device hands over, for every access-code match, the flagged bit and the bits that
 * followed it (wmb_frame).  This file turns one such candidate into a datagram, doing in
 * one pass over the bit list what the reference does bit by bit in
 *   t1_c1_packet_decoder.h:272-460 (per-bit handlers), :649-712 (driver, RSSI abort),
 *   :463-536 (block CRCs), :551-636 (CRC strip)   and   s1_packet_decoder.h:132-282.
 */
#include "wmb_framer.h"
#include "wmb_frame_a.h"

#include <stdio.h>
#include <string.h>
#include <sys/time.h>
#include <time.h>

#define CAPTURE_THRESHOLD 5u           /* PACKET_CAPTURE_THRESHOLD, t1_c1_packet_decoder.h:36 */

/* ---- CRC-16, polynomial 0x3D65 (t1_c1_packet_decoder.h:463-469) ---------------- */

static uint16_t g_crc_tab[256];
static int g_crc_ready;

static void crc_init(void)
{
    for (unsigned i = 0; i < 256; i++) {
        unsigned c = i << 8;
        for (int b = 0; b < 8; b++) c = (c & 0x8000u) ? ((c << 1) ^ 0x3D65u) : (c << 1);
        g_crc_tab[i] = (uint16_t)c;
    }
    g_crc_ready = 1;
}

uint16_t wmb_crc16(const uint8_t *data, size_t n)
{
    if (!g_crc_ready) crc_init();
    unsigned crc = 0;
    for (size_t i = 0; i < n; i++) crc = (g_crc_tab[data[i] ^ (crc >> 8)] ^ (crc << 8)) & 0xFFFFu;
    return (uint16_t)(~crc & 0xFFFFu);
}

static int block_ok(const uint8_t *p, size_t n)      /* n includes the two CRC bytes */
{
    if (n < 2) return 0;
    return wmb_crc16(p, n - 2) == (uint16_t)((p[n - 2] << 8) | p[n - 1]);
}

/* format A: 10-byte first block, 16-byte blocks after it (:471-506) */
static int crc_check_a(const uint8_t *p, size_t n)
{
    if (n < 12 || !block_ok(p, 12)) return 0;
    for (size_t off = 12; off < n;) {
        const size_t blk = (n - off >= 18) ? 18 : n - off;
        if (!block_ok(p + off, blk)) return 0;
        off += blk;
    }
    return 1;
}

/* format B: CRC over the first 126 bytes, then over the rest (:508-536); layout in wmb_frame_a.h */
static int crc_check_b(const uint8_t *p, size_t n)
{
    if (n < 12) return 0;
    for (uint32_t j = 0; j < wmb_nblk_b((uint32_t)n); j++)
        if (!block_ok(p + wmb_blk_off_b(j), wmb_blk_len_b((uint32_t)n, j))) return 0;
    return 1;
}

/* CRC strip, returns the stripped length (:551-592 format A, :595-636 format B) */
static unsigned strip_a(uint8_t *p, unsigned n)
{
    if (p[0] == 0 || n < 12) return 0;
    unsigned out = 10;
    for (unsigned off = 12; off < n;) {
        const unsigned blk = (n - off >= 18) ? 18 : n - off;
        memmove(p + out, p + off, blk - 2);
        out += blk - 2; off += blk;
    }
    return out;
}

static unsigned strip_b(uint8_t *p, unsigned n)
{
    if (p[0] < 2 || n < 12) return 0;
    unsigned out = 0;
    for (unsigned off = 0; off < n;) {
        const unsigned blk = (n - off >= 128) ? 128 : n - off;
        if (blk < 2) break;                       /* the reference reads out of bounds here */
        memmove(p + out, p + off, blk - 2);
        out += blk - 2; off += blk;
        p[0] = (uint8_t)(p[0] - 2);               /* :618, :630 */
    }
    return out;
}

/* ---- tables --------------------------------------------------------------------- */

/* EN 13757-4 3-out-of-6: code word -> nibble, 0xFF invalid (t1_c1_packet_decoder.h:50-65) */
static uint8_t nibble_3of6(unsigned c)
{
    static const int8_t tab[64] = {
        -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, 3, -1, 1, 2, -1,
        -1, -1, -1, 7, -1, -1, 0, -1, -1, 5, 6, -1, 4, -1, -1, -1,
        -1, -1, -1, 11, -1, 9, 10, -1, -1, 15, -1, -1, 8, -1, -1, -1,
        -1, 13, 14, -1, 12, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1 };
    const int v = tab[c & 63u];
    return v < 0 ? 0xFF : (uint8_t)v;
}

static unsigned wmb_tlg_length_format_a(unsigned L)      /* t1_c1_packet_decoder.h:68-96 */
{
    return 1 + L + 2 * (1 + (L > 9 ? (L - 9 + 15) / 16 : 0));
}

/* ---- bit cursor ----------------------------------------------------------------- */

typedef struct cursor {
    const wmb_frame *f;
    uint32_t pos;            /* index of the last consumed bit */
    int stop;                /* 0 running, WMB_DEC_ABORT+10 / WMB_DEC_NEED_MORE+10 */
} cursor;

enum { STOP_ABORT = 1, STOP_MORE = 2 };

/* Consume `n` bits MSB first.  After every bit except the telegram's very last one the
 * reference drops the packet when rssi < 5 (:703-710).  Returns 0 on success. */
static int take(cursor *c, unsigned n, int last_of_telegram, unsigned *value)
{
    unsigned v = 0;
    for (unsigned k = 0; k < n; k++) {
        if (c->pos + 1 >= c->f->nbits) { c->stop = STOP_MORE; return 1; }
        c->pos++;
        const wmb_bit w = c->f->bits[c->pos];
        v = (v << 1) | WMB_BIT_DATA(w);
        const int final_bit = last_of_telegram && k + 1 == n;
        if (!final_bit && WMB_BIT_RSSI(w) < CAPTURE_THRESHOLD) { c->stop = STOP_ABORT; return 1; }
    }
    *value = v;
    return 0;
}

static void finish(const cursor *c, wmb_decoded *d, const char *mode, uint8_t *pkt, unsigned len,
                   int bframe, unsigned err3of6)
{
    const wmb_bit last = c->f->bits[c->pos];
    d->status = WMB_DEC_LINE;
    d->consumed = c->pos + 1;
    d->end_sample = c->f->sync_sample + WMB_BIT_OFFSET(last);
    memcpy(d->mode, mode, 3);
    d->crc_ok = (uint8_t)(bframe ? crc_check_b(pkt, len) : crc_check_a(pkt, len));
    d->ok_3of6 = (uint8_t)(err3of6 ^ 1u);
    d->packet_rssi = WMB_BIT_RSSI(c->f->bits[1]);            /* rssi at the first bit after sync (:295) */
    d->current_rssi = WMB_BIT_RSSI(last);
    memcpy(&d->serial, pkt + 4, 4);                           /* get_serial(), :638-645 (host is LE) */
    d->len = bframe ? strip_b(pkt, len) : strip_a(pkt, len);
    memcpy(d->datagram, pkt, sizeof(d->datagram));
}

static void stopped(const cursor *c, wmb_decoded *d)
{
    d->status = (c->stop == STOP_MORE) ? WMB_DEC_NEED_MORE : WMB_DEC_ABORT;
    d->consumed = c->pos + 1;
    d->end_sample = c->f->sync_sample + WMB_BIT_OFFSET(c->f->bits[c->pos]);
}

/* ---- T1 and C1 ------------------------------------------------------------------ */

static void decode_t1c1(cursor *c, wmb_decoded *d)
{
    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    unsigned hi6, lo6, v;

    if (take(c, 6, 0, &hi6) || take(c, 6, 0, &lo6)) { stopped(c, d); return; }
    const unsigned hi = nibble_3of6(hi6), lo = nibble_3of6(lo6);
    const unsigned mode = (hi6 << 6) | lo6;

    if (hi != 0xFF && lo != 0xFF) {
        /* T1: 3-out-of-6 coded L-field and data (:298-392) */
        const unsigned L = (hi << 4) | lo;
        const unsigned len = wmb_tlg_length_format_a(L);
        unsigned err = 0, l = 0;
        pkt[l++] = (uint8_t)L;
        while (l < len) {
            const int last = (l + 1 >= len);
            if (take(c, 6, 0, &hi6) || take(c, 6, last, &lo6)) { stopped(c, d); return; }
            const unsigned h = nibble_3of6(hi6), lw = nibble_3of6(lo6);
            if (h == 0xFF || lw == 0xFF) err = 1;
            pkt[l++] = (uint8_t)((h == 0xFF ? 0xFFu : h << 4) | lw);
        }
        finish(c, d, "T1", pkt, len, 0, err);
        return;
    }
    if (mode != 0x54Cu && mode != 0x543u) {        /* neither L-field nor C1 mode word (:334-337) */
        c->stop = STOP_ABORT; stopped(c, d); return;
    }
    /* C1: 4-bit trailer, 8-bit L, NRZ bytes (:399-460) */
    const int bframe = (mode == 0x543u);
    if (take(c, 4, 0, &v)) { stopped(c, d); return; }
    if (v != 0xDu) { c->stop = STOP_ABORT; stopped(c, d); return; }
    if (take(c, 8, 0, &v)) { stopped(c, d); return; }
    const unsigned len = bframe ? 1 + v : wmb_tlg_length_format_a(v);
    unsigned l = 0;
    pkt[l++] = (uint8_t)v;
    do {
        const int last = (l + 1 >= len);
        if (take(c, 8, last, &v)) { stopped(c, d); return; }
        pkt[l++] = (uint8_t)v;
    } while (l < len);
    finish(c, d, "C1", pkt, len, bframe, 0);
}

/* ---- S1 ------------------------------------------------------------------------- */

/* one Manchester coded byte: 16 chips, "01" = 1, "10" = 0 (s1_packet_decoder.h:35-37, :152-168) */
static int take_manchester_byte(cursor *c, int last_of_telegram, unsigned *value)
{
    unsigned v = 0;
    for (int k = 0; k < 8; k++) {
        unsigned a, b;
        if (take(c, 1, 0, &a)) return 1;
        /* the violation check runs before the rssi check on the second chip */
        if (c->pos + 1 >= c->f->nbits) { c->stop = STOP_MORE; return 1; }
        c->pos++;
        const wmb_bit w = c->f->bits[c->pos];
        b = WMB_BIT_DATA(w);
        if (a == b) { c->stop = STOP_ABORT; return 1; }
        v = (v << 1) | b;
        const int final_bit = last_of_telegram && k == 7;
        if (!final_bit && WMB_BIT_RSSI(w) < CAPTURE_THRESHOLD) { c->stop = STOP_ABORT; return 1; }
    }
    *value = v;
    return 0;
}

static void decode_s1(cursor *c, wmb_decoded *d)
{
    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    unsigned v;
    if (take_manchester_byte(c, 0, &v)) { stopped(c, d); return; }
    const unsigned len = wmb_tlg_length_format_a(v);
    unsigned l = 0;
    pkt[l++] = (uint8_t)v;
    while (l < len) {
        const int last = (l + 1 >= len);
        if (take_manchester_byte(c, last, &v)) { stopped(c, d); return; }
        pkt[l++] = (uint8_t)v;
    }
    finish(c, d, "S1", pkt, len, 0, 0);
}

void wmb_frame_decode(const wmb_frame *f, wmb_decoded *d)
{
    memset(d, 0, sizeof(*d));
    cursor c = { f, 0, 0 };
    if (f->nbits == 0) { d->status = WMB_DEC_NEED_MORE; return; }
    /* the flagged bit itself: idle handler keeps the state, then the rssi check (:703-710) */
    if (WMB_BIT_RSSI(f->bits[0]) < CAPTURE_THRESHOLD) { c.stop = STOP_ABORT; stopped(&c, d); return; }
    if (f->chain == WMB_CHAIN_T1C1) decode_t1c1(&c, d);
    else decode_s1(&c, d);
}

/* ---- erasure repair (definition in wmbus_b200_framer.h; device twin: K4R, wmb_kernels.cuh) ------- */

#define REP_MAX_ERASURES 3u

typedef struct erasure {
    unsigned byte, shift, n;            /* the byte, where the filling goes in it, how many fillings */
    uint8_t  fill[6];
} erasure;

/* the code words at Hamming distance 1 from a 6-bit word, lowest flipped bit first: 2..4 of them for an invalid word of
 * weight 2 or 4, none for weight 0, 1, 5, 6 or an invalid word of weight 3 */
static unsigned fillings_3of6(unsigned w, uint8_t *fill)
{
    unsigned n = 0;
    for (unsigned k = 0; k < 6; k++) {
        const unsigned v = nibble_3of6(w ^ (1u << k));
        if (v != 0xFFu) fill[n++] = (uint8_t)v;
    }
    return n;
}

static unsigned bits_at(const wmb_bit *b, unsigned first, unsigned n)      /* MSB first */
{
    unsigned v = 0;
    for (unsigned k = 0; k < n; k++) v = (v << 1) | WMB_BIT_DATA(b[first + k]);
    return v;
}

int wmb_frame_repair(const wmb_frame *f, uint32_t e_max, wmb_repaired *out)
{
    memset(out, 0, sizeof(*out));
    if (e_max > REP_MAX_ERASURES) return WMB_E_INVAL;
    if (e_max == 0 || f->nbits == 0) return WMB_OK;
    const wmb_bit *b = f->bits;
    const int t1 = f->chain == WMB_CHAIN_T1C1;

    /* candidates: a line whose CRCs fail, an S1 abort on a Manchester violation after the L-field byte */
    wmb_decoded d;
    wmb_frame_decode(f, &d);
    if (d.status == WMB_DEC_LINE && !d.crc_ok) {
        out->had_line = 1;
        if (d.mode[0] == 'C') { out->outcome = WMB_REP_UNREPAIRABLE; return WMB_OK; }     /* NRZ: no erasures */
    } else if (d.status == WMB_DEC_ABORT && !t1) {
        const unsigned pos = d.consumed - 1;
        if (pos < 18 || (pos & 1u) || WMB_BIT_DATA(b[pos]) != WMB_BIT_DATA(b[pos - 1])) return WMB_OK;
    } else return WMB_OK;

    unsigned L = 0;
    if (t1) L = (nibble_3of6(bits_at(b, 1, 6)) << 4) | nibble_3of6(bits_at(b, 7, 6));
    else for (unsigned k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(b[2 + 2 * k]);
    const unsigned len = wmb_tlg_length_format_a(L);
    const unsigned P = 1 + (t1 ? 12u : 16u) * len;
    if (f->nbits < P) { out->outcome = WMB_REP_TRUNCATED; return WMB_OK; }
    if (len < 12) { out->outcome = WMB_REP_UNREPAIRABLE; return WMB_OK; }
    for (unsigned i = 0; i + 1 < P; i++)
        if (WMB_BIT_RSSI(b[i]) < CAPTURE_THRESHOLD) { out->outcome = WMB_REP_UNREPAIRABLE; return WMB_OK; }

    /* the received bytes with their erasures zeroed, and the erasures in chip order */
    uint8_t pkt[292];
    static __thread erasure er[8 * 292];
    unsigned ner = 0;
    memset(pkt, 0, sizeof(pkt));
    pkt[0] = (uint8_t)L;
    for (unsigned l = 1; l < len; l++) {
        unsigned v = 0;
        if (t1) {
            for (unsigned s = 0; s < 2; s++) {
                const unsigned w = bits_at(b, 1 + 12 * l + 6 * s, 6), shift = s ? 0u : 4u, nib = nibble_3of6(w);
                if (nib != 0xFFu) { v |= nib << shift; continue; }
                erasure *e = &er[ner++];
                e->byte = l; e->shift = shift; e->n = fillings_3of6(w, e->fill);
                if (!e->n) { out->outcome = WMB_REP_UNREPAIRABLE; return WMB_OK; }
            }
        } else {
            for (unsigned k = 0; k < 8; k++) {
                const unsigned a = WMB_BIT_DATA(b[1 + 16 * l + 2 * k]), c = WMB_BIT_DATA(b[2 + 16 * l + 2 * k]);
                if (a != c) { v |= c << (7 - k); continue; }
                erasure *e = &er[ner++];
                e->byte = l; e->shift = 7 - k; e->n = 2; e->fill[0] = 0; e->fill[1] = 1;
            }
        }
        pkt[l] = (uint8_t)v;
    }
    const unsigned nblk = wmb_nblk_a(len);
    for (unsigned j = 0, k = 0; j < nblk; j++) {
        const unsigned off = wmb_blk_off_a(j), blk = wmb_blk_len_a(len, j);
        unsigned ne = 0;
        while (k < ner && er[k].byte < off + blk) { k++; ne++; }
        if (ne > e_max) { out->outcome = WMB_REP_TOO_MANY; return WMB_OK; }
    }

    /* block by block, in frame order: exactly one filling (mixed radix, the block's first erasure lowest) passes */
    unsigned k = 0, erasures = 0, blocks = 0;
    for (unsigned j = 0; j < nblk; j++) {
        const unsigned off = wmb_blk_off_a(j), blk = wmb_blk_len_a(len, j);
        unsigned nf = 1, pass = 0, first = 0;
        const erasure *e = &er[k];
        unsigned ne = 0;
        while (k < ner && er[k].byte < off + blk) { nf *= er[k].n; k++; ne++; }
        for (unsigned i = 0; i < nf; i++) {
            uint8_t q[18];
            memcpy(q, pkt + off, blk);
            for (unsigned m = 0, rest = i; m < ne; m++) {
                q[e[m].byte - off] |= (uint8_t)(e[m].fill[rest % e[m].n] << e[m].shift);
                rest /= e[m].n;
            }
            if (block_ok(q, blk)) { if (!pass) first = i; pass++; }
        }
        if (pass != 1) { out->outcome = pass ? WMB_REP_AMBIGUOUS : WMB_REP_UNREPAIRABLE; return WMB_OK; }
        for (unsigned m = 0, rest = first; m < ne; m++) {
            pkt[e[m].byte] |= (uint8_t)(e[m].fill[rest % e[m].n] << e[m].shift);
            rest /= e[m].n;
        }
        erasures += ne; blocks += ne ? 1u : 0u;
    }
    if (!erasures) { out->outcome = WMB_REP_UNREPAIRABLE; return WMB_OK; }

    const cursor c = { f, P - 1, 0 };
    finish(&c, &out->line, t1 ? "T1" : "S1", pkt, len, 0, 0);
    out->outcome = WMB_REP_REPAIRED;
    out->erasures = erasures;
    out->blocks = blocks;
    return WMB_OK;
}

/* ---- C1 soft repair (definition in wmbus_b200_framer.h; device twin: K4S, wmb_kernels.cuh) ------------------------ */

/* a before b in the search order: a bit without a value first, then lower r, then lower index */
static int soft_before(int sa, int64_t ra, unsigned ja, int sb, int64_t rb, unsigned jb)
{
    if (sa != sb) return sa < sb;
    if (ra != rb) return ra < rb;
    return ja < jb;
}

static void repair_soft_c1(const wmb_frame *f, const int16_t *soft, uint32_t k_max, wmb_repaired *out)
{
    const wmb_bit *b = f->bits;
    out->had_line = 1;
    out->outcome = WMB_REP_UNREPAIRABLE;
    const int bframe = bits_at(b, 1, 12) == 0x543u;
    const unsigned L = bits_at(b, 17, 8);
    const unsigned len = bframe ? 1 + L : wmb_tlg_length_format_a(L);
    const unsigned P = 17 + 8 * len;
    if (len < 12) return;

    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    for (unsigned l = 0; l < len; l++) pkt[l] = (uint8_t)bits_at(b, 17 + 8 * l, 8);
    int64_t n0 = 0, n1 = 0, s0 = 0, s1 = 0;
    for (unsigned j = 17; j < P; j++) {
        if (soft[j] == WMB_SOFT_NONE) continue;
        if (WMB_BIT_DATA(b[j])) { n1++; s1 += soft[j]; } else { n0++; s0 += soft[j]; }
    }
    /* r of bit j; has[j] = 0 for a bit without a value */
    static __thread int64_t r[8 * 292];
    static __thread int has[8 * 292];
    for (unsigned j = 17; j < P; j++) {
        const int64_t sign = WMB_BIT_DATA(b[j]) ? 1 : -1, v = soft[j];
        has[j - 17] = soft[j] != WMB_SOFT_NONE;
        r[j - 17] = !has[j - 17] ? 0 : n0 * n1 == 0 ? sign * v : sign * (v * 2 * n0 * n1 - (s1 * n0 + s0 * n1));
    }

    const unsigned nblk = bframe ? wmb_nblk_b(len) : wmb_nblk_a(len);
    unsigned flips = 0, blocks = 0;
    for (unsigned k = 0; k < nblk; k++) {
        const unsigned off = bframe ? wmb_blk_off_b(k) : wmb_blk_off_a(k), blk = bframe ? wmb_blk_len_b(len, k) : wmb_blk_len_a(len, k);
        if (block_ok(pkt + off, blk)) continue;
        /* the K least reliable flippable bits, by selection */
        const unsigned lo = 17 + 8 * (off ? off : 1), hi = 17 + 8 * (off + blk);
        const unsigned K = k_max < hi - lo ? k_max : hi - lo;
        unsigned sel[WMB_SOFT_K_MAX];
        for (unsigned t = 0; t < K; t++) {
            int found = 0;
            for (unsigned j = lo; j < hi; j++) {
                int taken = 0;
                for (unsigned u = 0; u < t; u++) taken |= sel[u] == j;
                if (taken) continue;
                if (!found || soft_before(has[j - 17], r[j - 17], j, has[sel[t] - 17], r[sel[t] - 17], sel[t])) { sel[t] = j; found = 1; }
            }
        }
        unsigned pass = 0, first = 0;
        for (unsigned x = 1; x < (1u << K); x++) {
            uint8_t q[128];
            memcpy(q, pkt + off, blk);
            for (unsigned t = 0; t < K; t++)
                if (x >> t & 1u) q[(sel[t] - 17) / 8 - off] ^= (uint8_t)(0x80u >> ((sel[t] - 17) % 8));
            if (block_ok(q, blk)) { if (!pass) first = x; pass++; }
        }
        if (pass != 1) { out->outcome = pass ? WMB_REP_AMBIGUOUS : WMB_REP_UNREPAIRABLE; return; }
        for (unsigned t = 0; t < K; t++)
            if (first >> t & 1u) { pkt[(sel[t] - 17) / 8] ^= (uint8_t)(0x80u >> ((sel[t] - 17) % 8)); flips++; }
        blocks++;
    }
    const cursor c = { f, P - 1, 0 };
    finish(&c, &out->line, "C1", pkt, len, bframe, 0);
    out->outcome = WMB_REP_REPAIRED;
    out->erasures = flips;
    out->blocks = blocks;
}

int wmb_frame_repair_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t k_max, wmb_repaired *out)
{
    if (k_max > WMB_SOFT_K_MAX || e_max > REP_MAX_ERASURES) { memset(out, 0, sizeof(*out)); return WMB_E_INVAL; }
    if (k_max && soft && f->nbits && f->chain == WMB_CHAIN_T1C1) {
        wmb_decoded d;
        wmb_frame_decode(f, &d);
        if (d.status == WMB_DEC_LINE && !d.crc_ok && d.mode[0] == 'C') {
            memset(out, 0, sizeof(*out));
            repair_soft_c1(f, soft, k_max, out);
            return WMB_OK;
        }
    }
    return wmb_frame_repair(f, e_max, out);
}

/* ---- T1 soft repair (definition in wmbus_b200_framer.h; device twin: K4S, wmb_kernels.cuh) ------------------------ */

static void repair_soft_t1(const wmb_frame *f, const int16_t *soft, uint32_t s_max, wmb_repaired *out)
{
    const wmb_bit *b = f->bits;
    const unsigned L = (nibble_3of6(bits_at(b, 1, 6)) << 4) | nibble_3of6(bits_at(b, 7, 6));
    const unsigned len = wmb_tlg_length_format_a(L), P = 1 + 12 * len, nsym = 2 * len;
    int64_t n0 = 0, n1 = 0, s0 = 0, s1 = 0;
    for (unsigned j = 13; j < P; j++) {
        if (soft[j] == WMB_SOFT_NONE) continue;
        if (WMB_BIT_DATA(b[j])) { n1++; s1 += soft[j]; } else { n0++; s0 += soft[j]; }
    }
    /* per symbol i (byte i / 2, the high nibble first): hard nibble (0xFF invalid), ML, runner-up, delta, has values */
    static __thread uint8_t hard[2 * 292], ml[2 * 292], ru[2 * 292];
    static __thread int64_t delta[2 * 292];
    static __thread int has[2 * 292];
    for (unsigned i = 2; i < nsym; i++) {
        int64_t y[6];
        has[i] = 1;
        for (unsigned c = 0; c < 6; c++) {
            const unsigned j = 1 + 6 * i + c;
            const int64_t v = soft[j];
            if (soft[j] == WMB_SOFT_NONE) { has[i] = 0; y[c] = 0; }
            else y[c] = n0 * n1 == 0 ? v : v * 2 * n0 * n1 - (s1 * n0 + s0 * n1);
        }
        uint32_t m, r;
        wmb_t1_sym_ml(y, &m, &r, &delta[i]);
        ml[i] = (uint8_t)m; ru[i] = (uint8_t)r;
        hard[i] = nibble_3of6(bits_at(b, 1 + 6 * i, 6));
    }

    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    pkt[0] = (uint8_t)L;
    for (unsigned l = 1; l < len; l++) pkt[l] = (uint8_t)(((hard[2 * l] & 15u) << 4) | (hard[2 * l + 1] & 15u));
    unsigned changed = 0, blocks = 0;
    for (unsigned k = 0; k < wmb_nblk_a(len); k++) {
        const unsigned off = wmb_blk_off_a(k), blk = wmb_blk_len_a(len, k);
        const unsigned lo = 2 * (off ? off : 1), hi = 2 * (off + blk);    /* the block's searchable symbols */
        int valid = 1;
        for (unsigned i = lo; i < hi; i++) valid &= hard[i] != 0xFFu;
        if (valid && block_ok(pkt + off, blk)) continue;
        for (unsigned i = lo; i < hi; i++) pkt[i / 2] = (uint8_t)(i & 1u ? (pkt[i / 2] & 0xF0u) | ml[i] : (pkt[i / 2] & 0x0Fu) | ml[i] << 4);
        /* the K symbols of lowest delta, by selection (a symbol with a chip without a value first, ties: lower index) */
        const unsigned K = s_max < hi - lo ? s_max : hi - lo;
        unsigned sel[WMB_SOFT_K_MAX];
        for (unsigned t = 0; t < K; t++) {
            int found = 0;
            for (unsigned i = lo; i < hi; i++) {
                int taken = 0;
                for (unsigned u = 0; u < t; u++) taken |= sel[u] == i;
                if (taken) continue;
                if (!found || soft_before(has[i], delta[i], i, has[sel[t]], delta[sel[t]], sel[t])) { sel[t] = i; found = 1; }
            }
        }
        unsigned pass = 0, first = 0;
        for (unsigned x = 0; x < (1u << K); x++) {
            uint8_t q[18];
            memcpy(q, pkt + off, blk);
            for (unsigned t = 0; t < K; t++)
                if (x >> t & 1u) q[sel[t] / 2 - off] ^= (uint8_t)((ml[sel[t]] ^ ru[sel[t]]) << (sel[t] & 1u ? 0 : 4));
            if (block_ok(q, blk)) { if (!pass) first = x; pass++; }
        }
        if (pass != 1) { out->outcome = pass ? WMB_REP_AMBIGUOUS : WMB_REP_UNREPAIRABLE; return; }
        for (unsigned t = 0; t < K; t++)
            if (first >> t & 1u) pkt[sel[t] / 2] ^= (uint8_t)((ml[sel[t]] ^ ru[sel[t]]) << (sel[t] & 1u ? 0 : 4));
        for (unsigned i = lo; i < hi; i++) changed += hard[i] != (i & 1u ? pkt[i / 2] & 15u : pkt[i / 2] >> 4);
        blocks++;
    }
    const cursor c = { f, P - 1, 0 };
    finish(&c, &out->line, "T1", pkt, len, 0, 0);
    out->outcome = WMB_REP_REPAIRED;
    out->erasures = changed < 255 ? changed : 255;         /* the device record's byte */
    out->blocks = blocks;
}

int wmb_frame_repair_t1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    if (s_max > WMB_SOFT_K_MAX || e_max > REP_MAX_ERASURES) { memset(out, 0, sizeof(*out)); return WMB_E_INVAL; }
    const int rc = wmb_frame_repair(f, e_max, out);
    if (rc || !s_max || !soft || f->chain != WMB_CHAIN_T1C1) return rc;
    if (out->outcome != WMB_REP_TOO_MANY && out->outcome != WMB_REP_UNREPAIRABLE) return rc;
    wmb_decoded d;
    wmb_frame_decode(f, &d);
    if (d.status != WMB_DEC_LINE || d.crc_ok || d.mode[0] != 'T') return rc;
    /* a line reaches P and has no rssi drop before P - 1; len >= 12 is the rule's own */
    const unsigned L = (nibble_3of6(bits_at(f->bits, 1, 6)) << 4) | nibble_3of6(bits_at(f->bits, 7, 6));
    if (wmb_tlg_length_format_a(L) < 12) return rc;
    memset(out, 0, sizeof(*out));
    out->had_line = 1;
    repair_soft_t1(f, soft, s_max, out);
    return WMB_OK;
}

/* ---- S1 soft repair (definition in wmbus_b200_framer.h; device twin: K4S, wmb_kernels.cuh) ------------------------ */

static unsigned s1_bit(const uint8_t *pkt, unsigned p) { return pkt[p / 8] >> (7 - p % 8) & 1u; }

static void repair_soft_s1(const wmb_frame *f, const int16_t *soft, unsigned L, uint32_t s_max, wmb_repaired *out)
{
    const wmb_bit *b = f->bits;
    const unsigned len = wmb_tlg_length_format_a(L), npair = 8 * len;
    /* per pair p = 8 l + bit: hard bit (2: a violation), ML bit, search key */
    static __thread uint8_t hard[8 * 292], ml[8 * 292];
    static __thread uint32_t key[8 * 292];
    for (unsigned p = 8; p < npair; p++) {
        const unsigned a = WMB_BIT_DATA(b[1 + 2 * p]), c = WMB_BIT_DATA(b[2 + 2 * p]);
        uint32_t m;
        key[p] = wmb_s1_pair(soft[1 + 2 * p], soft[2 + 2 * p], a, c, p, &m);
        ml[p] = (uint8_t)m;
        hard[p] = (uint8_t)(a != c ? c : 2u);
    }

    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    pkt[0] = (uint8_t)L;
    for (unsigned p = 8; p < npair; p++) pkt[p / 8] |= (uint8_t)((hard[p] & 1u) << (7 - p % 8));
    unsigned changed = 0, blocks = 0;
    for (unsigned k = 0; k < wmb_nblk_a(len); k++) {
        const unsigned off = wmb_blk_off_a(k), blk = wmb_blk_len_a(len, k);
        const unsigned lo = 8 * (off ? off : 1), hi = 8 * (off + blk);    /* the block's searchable pairs */
        int valid = 1;
        for (unsigned p = lo; p < hi; p++) valid &= hard[p] != 2u;
        if (valid && block_ok(pkt + off, blk)) continue;
        for (unsigned p = lo; p < hi; p++) pkt[p / 8] = (uint8_t)((pkt[p / 8] & ~(0x80u >> p % 8)) | ml[p] << (7 - p % 8));
        /* the K pairs of lowest key, by selection (keys are unique) */
        const unsigned K = s_max < hi - lo ? s_max : hi - lo;
        unsigned sel[WMB_SOFT_K_MAX];
        for (unsigned t = 0; t < K; t++) {
            uint32_t best = 0xFFFFFFFFu;
            for (unsigned p = lo; p < hi; p++)
                if (key[p] < best && (t == 0 || key[p] > key[sel[t - 1]])) { best = key[p]; sel[t] = p; }
        }
        unsigned pass = 0, first = 0;
        for (unsigned x = 0; x < (1u << K); x++) {
            uint8_t q[18];
            memcpy(q, pkt + off, blk);
            for (unsigned t = 0; t < K; t++)
                if (x >> t & 1u) q[sel[t] / 8 - off] ^= (uint8_t)(0x80u >> sel[t] % 8);
            if (block_ok(q, blk)) { if (!pass) first = x; pass++; }
        }
        if (pass != 1) { out->outcome = pass ? WMB_REP_AMBIGUOUS : WMB_REP_UNREPAIRABLE; return; }
        for (unsigned t = 0; t < K; t++)
            if (first >> t & 1u) pkt[sel[t] / 8] ^= (uint8_t)(0x80u >> sel[t] % 8);
        for (unsigned p = lo; p < hi; p++) changed += hard[p] != s1_bit(pkt, p);
        blocks++;
    }
    const cursor c = { f, 16 * len, 0 };
    finish(&c, &out->line, "S1", pkt, len, 0, 0);
    out->outcome = WMB_REP_REPAIRED;
    out->erasures = changed < 255 ? changed : 255;         /* the device record's byte */
    out->blocks = blocks;
}

int wmb_frame_repair_s1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    if (s_max > WMB_SOFT_K_MAX || e_max > REP_MAX_ERASURES) { memset(out, 0, sizeof(*out)); return WMB_E_INVAL; }
    const int rc = wmb_frame_repair(f, e_max, out);
    if (rc || !s_max || !soft || f->chain != WMB_CHAIN_S1) return rc;
    /* TOO_MANY / UNREPAIRABLE: a candidate of the erasure rule (a line with crc_ok = 0 or a violation abort) whose list
     * reaches P; UNREPAIRABLE also stands for len < 12 and an rssi drop, which stay so */
    if (out->outcome != WMB_REP_TOO_MANY && out->outcome != WMB_REP_UNREPAIRABLE) return rc;
    unsigned L = 0;
    for (unsigned k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(f->bits[2 + 2 * k]);
    const unsigned len = wmb_tlg_length_format_a(L), P = 1 + 16 * len;
    if (len < 12) return rc;
    for (unsigned i = 0; i + 1 < P; i++)
        if (WMB_BIT_RSSI(f->bits[i]) < CAPTURE_THRESHOLD) return rc;
    const uint32_t had_line = out->had_line;
    memset(out, 0, sizeof(*out));
    out->had_line = had_line;
    out->outcome = WMB_REP_UNREPAIRABLE;
    repair_soft_s1(f, soft, L, s_max, out);
    return WMB_OK;
}

/* ---- output --------------------------------------------------------------------- */

void wmb_make_time_string(char *ts, size_t n)
{
    /* the calendar part only changes once a second: localtime_r/strftime are redone when tv_sec moves */
    static __thread time_t cached_sec = (time_t)-1;
    static __thread char cached_fmt[64];
    struct timeval tv;
    if (gettimeofday(&tv, NULL) != 0) { if (n) ts[0] = 0; return; }
    if (tv.tv_sec != cached_sec) {
        struct tm tmv;
        if (localtime_r(&tv.tv_sec, &tmv) == NULL) { if (n) ts[0] = 0; return; }
        strftime(cached_fmt, sizeof(cached_fmt), "%Y-%m-%d %H:%M:%S.", &tmv);
        cached_sec = tv.tv_sec;
    }
    const size_t l = strlen(cached_fmt);
    if (n < l + 7) { if (n) ts[0] = 0; return; }
    memcpy(ts, cached_fmt, l);
    unsigned us = (unsigned)tv.tv_usec;
    for (int i = 5; i >= 0; i--) { ts[l + (size_t)i] = (char)('0' + us % 10u); us /= 10u; }
    ts[l + 6] = 0;
}

static size_t put_str(char *buf, size_t len, size_t cap, const char *s)
{
    while (*s && len + 1 < cap) buf[len++] = *s++;
    return len;
}

static size_t put_u32(char *buf, size_t len, size_t cap, uint32_t v)
{
    char tmp[10];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10u); v /= 10u; } while (v);
    while (n && len + 1 < cap) buf[len++] = tmp[--n];
    return len;
}

/* hand-rolled (no printf machinery): a batch can carry thousands of lines */
size_t wmb_format_line(const wmb_decoded *d, const char *algo_prefix, const char *timestamp,
                       char *buf, size_t cap)
{
    static const char hexd[] = "0123456789abcdef", hexu[] = "0123456789ABCDEF";
    if (cap < 2) return 0;
    size_t len = 0;
    if (algo_prefix) len = put_str(buf, len, cap, algo_prefix);
    len = put_str(buf, len, cap, d->mode);
    if (len + 1 < cap) buf[len++] = ';';
    len = put_u32(buf, len, cap, d->crc_ok);
    if (len + 1 < cap) buf[len++] = ';';
    len = put_u32(buf, len, cap, d->ok_3of6);
    if (len + 1 < cap) buf[len++] = ';';
    len = put_str(buf, len, cap, timestamp);
    if (len + 1 < cap) buf[len++] = ';';
    len = put_u32(buf, len, cap, d->packet_rssi);
    if (len + 1 < cap) buf[len++] = ';';
    len = put_u32(buf, len, cap, d->current_rssi);
    if (len + 1 < cap) buf[len++] = ';';
    for (int sh = 28; sh >= 0 && len + 1 < cap; sh -= 4) buf[len++] = hexu[(d->serial >> sh) & 15u];   /* %08X */
    len = put_str(buf, len, cap, ";0x");
    for (uint32_t i = 0; i < d->len && len + 3 < cap; i++) {
        buf[len++] = hexd[d->datagram[i] >> 4];
        buf[len++] = hexd[d->datagram[i] & 15];
    }
    if (len + 1 < cap) buf[len++] = '\n';
    buf[len] = 0;
    return len;
}
