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
#include <stdlib.h>
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

/* ---- soft repair of C1, T1 and S1 (definitions in wmbus_b200_framer.h; device twin: K4S, wmb_kernels.cuh) ------------ */

/* One searchable unit: a C1 bit, a T1 symbol or an S1 pair.  Unit i of a code with W units per byte lies in byte i / W;
 * its value is (pkt[byte] >> shift) & mask. */
typedef struct soft_unit {
    uint64_t key;                /* the rule's search order as one integer, packed as K4S packs it: unique, lowest first */
    uint16_t byte;
    uint8_t  shift, mask;
    uint8_t  hard, ml, flip;     /* hard value (0xFF: invalid), ML value, ML ^ the alternative */
} soft_unit;

static __thread soft_unit g_units[8 * 292];

/* the centring of the soft values of chips [j0, P): y = v 2 n0 n1 - (S1 n0 + S0 n1), or v when one side is empty */
static void centring(const wmb_frame *f, const int16_t *soft, unsigned j0, unsigned P, int64_t *a, int64_t *t)
{
    int64_t n0 = 0, n1 = 0, s0 = 0, s1 = 0;
    for (unsigned j = j0; j < P; j++) {
        if (soft[j] == WMB_SOFT_NONE) continue;
        if (WMB_BIT_DATA(f->bits[j])) { n1++; s1 += soft[j]; } else { n0++; s0 += soft[j]; }
    }
    *a = 2 * n0 * n1;
    *t = s1 * n0 + s0 * n1;
}

/* C1 bit i = 8 l + k is frame bit 17 + i; key (has a value, r, 17 + i): |r| < 2^38 */
static void units_c1(const wmb_frame *f, const int16_t *soft, unsigned len, soft_unit *u)
{
    int64_t a, t;
    centring(f, soft, 17, 17 + 8 * len, &a, &t);
    for (unsigned i = 8; i < 8 * len; i++) {
        const unsigned j = 17 + i, bit = WMB_BIT_DATA(f->bits[j]);
        const int64_t v = soft[j], r = (bit ? 1 : -1) * (a == 0 ? v : v * a - t);
        const uint64_t key = v == WMB_SOFT_NONE ? j : (uint64_t)(r + ((int64_t)1 << 40)) << 12 | j;
        u[i] = (soft_unit){ key, (uint16_t)(i / 8), (uint8_t)(7 - i % 8), 1, (uint8_t)bit, (uint8_t)bit, 1 };
    }
}

/* T1 symbol i = 2 l + s (the high nibble first), chips 1 + 6 i ..; key (all chips have values, delta, i): delta < 2^43 */
static void units_t1(const wmb_frame *f, const int16_t *soft, unsigned len, soft_unit *u)
{
    int64_t a, t;
    centring(f, soft, 13, 1 + 12 * len, &a, &t);
    for (unsigned i = 2; i < 2 * len; i++) {
        int64_t y[6], delta;
        uint64_t has = 1;
        for (unsigned c = 0; c < 6; c++) {
            const int64_t v = soft[1 + 6 * i + c];
            if (v == WMB_SOFT_NONE) has = 0;
            y[c] = v == WMB_SOFT_NONE ? 0 : a == 0 ? v : v * a - t;
        }
        uint32_t ml, ru;
        wmb_t1_sym_ml(y, &ml, &ru, &delta);
        u[i] = (soft_unit){ has << 53 | (uint64_t)delta << 10 | i, (uint16_t)(i / 2), (uint8_t)(i & 1u ? 0 : 4), 15,
                            nibble_3of6(bits_at(f->bits, 1 + 6 * i, 6)), (uint8_t)ml, (uint8_t)(ml ^ ru) };
    }
}

/* S1 pair p = 8 l + k, chips 1 + 2 p and 2 + 2 p; key wmb_s1_pair's */
static void units_s1(const wmb_frame *f, const int16_t *soft, unsigned len, soft_unit *u)
{
    for (unsigned p = 8; p < 8 * len; p++) {
        const unsigned a = WMB_BIT_DATA(f->bits[1 + 2 * p]), c = WMB_BIT_DATA(f->bits[2 + 2 * p]);
        uint32_t ml;
        const uint32_t key = wmb_s1_pair(soft[1 + 2 * p], soft[2 + 2 * p], a, c, p, &ml);
        u[p] = (soft_unit){ key, (uint16_t)(p / 8), (uint8_t)(7 - p % 8), 1, (uint8_t)(a != c ? c : 0xFFu), (uint8_t)ml, 1 };
    }
}

/* The block search of the three rules over the units u[W .. W len) of a telegram with L-field L, whose list ends at
 * P - 1: per block, in frame order, the block's searchable units take their ML values, the K = min(k_max, units)
 * lowest keys are chosen, and exactly one of the 2^K patterns of alternatives must pass the block's CRC.
 *   - Pattern 0 is tried for C1 too: a C1 unit's ML value is its hard bit, so pattern 0 is the received block, which
 *     failed its CRC.
 *   - erasures counts the units whose final value differs from the hard one; for C1 that is the number of flipped bits
 *     (ML = hard), at most 6 per block and 17 blocks, below the device record's byte.
 *   - A frame B block is up to 128 bytes long, hence the trial buffer's size. */
static void soft_search(const wmb_frame *f, const soft_unit *u, unsigned W, unsigned L, unsigned len, int bframe,
                        unsigned P, uint32_t k_max, const char *mode, wmb_repaired *out)
{
    uint8_t pkt[292];
    memset(pkt, 0, sizeof(pkt));
    pkt[0] = (uint8_t)L;
    for (unsigned i = W; i < W * len; i++)
        if (u[i].hard != 0xFFu) pkt[u[i].byte] |= (uint8_t)(u[i].hard << u[i].shift);
    const unsigned nblk = bframe ? wmb_nblk_b(len) : wmb_nblk_a(len);
    unsigned changed = 0, blocks = 0;
    for (unsigned k = 0; k < nblk; k++) {
        const unsigned off = bframe ? wmb_blk_off_b(k) : wmb_blk_off_a(k), blk = bframe ? wmb_blk_len_b(len, k) : wmb_blk_len_a(len, k);
        const unsigned lo = W * (off ? off : 1), hi = W * (off + blk);        /* the block's searchable units */
        int valid = 1;
        for (unsigned i = lo; i < hi; i++) valid &= u[i].hard != 0xFFu;
        if (valid && block_ok(pkt + off, blk)) continue;
        for (unsigned i = lo; i < hi; i++)
            pkt[u[i].byte] = (uint8_t)((pkt[u[i].byte] & ~(u[i].mask << u[i].shift)) | u[i].ml << u[i].shift);
        /* the K units of lowest key, by selection */
        const unsigned K = k_max < hi - lo ? k_max : hi - lo;
        unsigned sel[WMB_SOFT_K_MAX];
        for (unsigned t = 0; t < K; t++) {
            uint64_t best = UINT64_MAX;
            for (unsigned i = lo; i < hi; i++)
                if (u[i].key < best && (t == 0 || u[i].key > u[sel[t - 1]].key)) { best = u[i].key; sel[t] = i; }
        }
        unsigned pass = 0, first = 0;
        for (unsigned x = 0; x < (1u << K); x++) {
            uint8_t q[128];
            memcpy(q, pkt + off, blk);
            for (unsigned t = 0; t < K; t++)
                if (x >> t & 1u) q[u[sel[t]].byte - off] ^= (uint8_t)(u[sel[t]].flip << u[sel[t]].shift);
            if (block_ok(q, blk)) { if (!pass) first = x; pass++; }
        }
        if (pass != 1) { out->outcome = pass ? WMB_REP_AMBIGUOUS : WMB_REP_UNREPAIRABLE; return; }
        for (unsigned t = 0; t < K; t++)
            if (first >> t & 1u) pkt[u[sel[t]].byte] ^= (uint8_t)(u[sel[t]].flip << u[sel[t]].shift);
        for (unsigned i = lo; i < hi; i++) changed += u[i].hard != (pkt[u[i].byte] >> u[i].shift & u[i].mask);
        blocks++;
    }
    const cursor c = { f, P - 1, 0 };
    finish(&c, &out->line, mode, pkt, len, bframe, 0);
    out->outcome = WMB_REP_REPAIRED;
    out->erasures = changed < 255 ? changed : 255;         /* the device record's byte */
    out->blocks = blocks;
}

/* a T1 / C1 line (mode[0] == m) whose CRCs fail */
static int crc_failed_line(const wmb_frame *f, char m)
{
    wmb_decoded d;
    wmb_frame_decode(f, &d);
    return d.status == WMB_DEC_LINE && !d.crc_ok && d.mode[0] == m;
}

/* the soft rules' own condition: len >= 12 and no rssi drop before P - 1 (a line has none) */
static int soft_candidate(const wmb_frame *f, unsigned len, unsigned P)
{
    if (len < 12) return 0;
    for (unsigned i = 0; i + 1 < P; i++)
        if (WMB_BIT_RSSI(f->bits[i]) < CAPTURE_THRESHOLD) return 0;
    return 1;
}

/* C1: a line with CRC errors, before the erasure rule (which finds it UNREPAIRABLE) */
int wmb_frame_repair_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t k_max, wmb_repaired *out)
{
    if (k_max > WMB_SOFT_K_MAX || e_max > REP_MAX_ERASURES) { memset(out, 0, sizeof(*out)); return WMB_E_INVAL; }
    if (!k_max || !soft || !f->nbits || f->chain != WMB_CHAIN_T1C1 || !crc_failed_line(f, 'C'))
        return wmb_frame_repair(f, e_max, out);
    memset(out, 0, sizeof(*out));
    out->had_line = 1;
    out->outcome = WMB_REP_UNREPAIRABLE;
    const int bframe = bits_at(f->bits, 1, 12) == 0x543u;
    const unsigned L = bits_at(f->bits, 17, 8), len = bframe ? 1 + L : wmb_tlg_length_format_a(L), P = 17 + 8 * len;
    if (!soft_candidate(f, len, P)) return WMB_OK;
    units_c1(f, soft, len, g_units);
    soft_search(f, g_units, 8, L, len, bframe, P, k_max, "C1", out);
    return WMB_OK;
}

/* T1 and S1: a candidate the erasure rule ends TOO_MANY or UNREPAIRABLE (T1: a line with CRC errors; S1: also a violation
 * abort), whose had_line stays; UNREPAIRABLE also stands for len < 12 and an rssi drop, which stay so */
static int repair_soft_after_erasures(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, int chain,
                                      wmb_repaired *out)
{
    if (s_max > WMB_SOFT_K_MAX || e_max > REP_MAX_ERASURES) { memset(out, 0, sizeof(*out)); return WMB_E_INVAL; }
    const int rc = wmb_frame_repair(f, e_max, out);
    if (rc || !s_max || !soft || f->chain != chain) return rc;
    if (out->outcome != WMB_REP_TOO_MANY && out->outcome != WMB_REP_UNREPAIRABLE) return rc;
    const int t1 = chain == WMB_CHAIN_T1C1;
    if (t1 && !crc_failed_line(f, 'T')) return rc;
    unsigned L = 0;
    if (t1) L = (nibble_3of6(bits_at(f->bits, 1, 6)) << 4) | nibble_3of6(bits_at(f->bits, 7, 6));
    else for (unsigned k = 0; k < 8; k++) L = (L << 1) | WMB_BIT_DATA(f->bits[2 + 2 * k]);
    const unsigned len = wmb_tlg_length_format_a(L), P = 1 + (t1 ? 12u : 16u) * len;
    if (!soft_candidate(f, len, P)) return rc;
    const uint32_t had_line = out->had_line;
    memset(out, 0, sizeof(*out));
    out->had_line = had_line;
    (t1 ? units_t1 : units_s1)(f, soft, len, g_units);
    soft_search(f, g_units, t1 ? 2 : 8, L, len, 0, P, s_max, t1 ? "T1" : "S1", out);
    return WMB_OK;
}

int wmb_frame_repair_t1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    return repair_soft_after_erasures(f, soft, e_max, s_max, WMB_CHAIN_T1C1, out);
}

int wmb_frame_repair_s1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out)
{
    return repair_soft_after_erasures(f, soft, e_max, s_max, WMB_CHAIN_S1, out);
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

/* ---- telegrams: one record per transmission (include/wmbus_b200_framer.h) ------------------------------------------ */

typedef struct tlg_cand {
    uint64_t sync;
    const wmb_decoded *d;       /* the line, or the repaired line                                               */
    size_t idx;                 /* input position: lines first, then repair records                             */
    uint8_t chain, src, verified;
} tlg_cand;

typedef struct tlg_rec {
    wmb_telegram t;
    const wmb_decoded *d;       /* the first candidate that carries the datagram; NULL when decoded = 0          */
} tlg_rec;

static int tlg_cand_cmp(const void *pa, const void *pb)
{
    const tlg_cand *a = (const tlg_cand *)pa, *b = (const tlg_cand *)pb;
    if (a->chain != b->chain) return a->chain < b->chain ? -1 : 1;
    if (a->sync != b->sync) return a->sync < b->sync ? -1 : 1;
    return a->idx < b->idx ? -1 : a->idx > b->idx;
}

/* (sync_sample, chain), then (mode, len, bytes) inside a group */
static int tlg_rec_cmp(const void *pa, const void *pb)
{
    const tlg_rec *a = (const tlg_rec *)pa, *b = (const tlg_rec *)pb;
    if (a->t.sync_sample != b->t.sync_sample) return a->t.sync_sample < b->t.sync_sample ? -1 : 1;
    if (a->t.chain != b->t.chain) return a->t.chain < b->t.chain ? -1 : 1;
    const int m = strncmp(a->t.mode, b->t.mode, sizeof(a->t.mode));
    if (m) return m;
    if (a->t.len != b->t.len) return a->t.len < b->t.len ? -1 : 1;
    return a->t.len ? memcmp(a->d->datagram, b->d->datagram, a->t.len) : 0;
}

static int same_datagram(const wmb_decoded *a, const wmb_decoded *b)
{
    return strncmp(a->mode, b->mode, sizeof(a->mode)) == 0 && a->len == b->len && memcmp(a->datagram, b->datagram, a->len) == 0;
}

/* point 4: the link-layer header fields the datagram is long enough for */
static void tlg_header(wmb_telegram *t, const uint8_t *p, unsigned len)
{
    if (len >= 1) { t->l = p[0]; t->valid |= WMB_TLG_F_L; }
    if (len >= 2) { t->c = p[1]; t->valid |= WMB_TLG_F_C; }
    if (len >= 4) {
        t->m = (uint16_t)(p[2] | p[3] << 8);
        t->manuf[0] = (char)(((t->m >> 10) & 31) + 64);
        t->manuf[1] = (char)(((t->m >> 5) & 31) + 64);
        t->manuf[2] = (char)((t->m & 31) + 64);
        t->valid |= WMB_TLG_F_M;
    }
    if (len >= 8) { t->id = (uint32_t)p[4] | (uint32_t)p[5] << 8 | (uint32_t)p[6] << 16 | (uint32_t)p[7] << 24; t->valid |= WMB_TLG_F_ID; }
    if (len >= 9) { t->version = p[8]; t->valid |= WMB_TLG_F_VERSION; }
    if (len >= 10) { t->type = p[9]; t->valid |= WMB_TLG_F_TYPE; }
    if (len >= 11) { t->ci = p[10]; t->valid |= WMB_TLG_F_CI; }
}

int wmb_group_telegrams(const wmb_line_info *info, const wmb_decoded *line, size_t n_lines,
                        const wmb_repair_record *repairs, size_t n_repairs,
                        wmb_telegram *out, size_t cap, uint8_t *data, size_t data_cap, size_t *n)
{
    static const uint64_t W[2] = { WMB_TLG_W_T1C1, WMB_TLG_W_S1 };
    if (!n || (n_lines && (!info || !line)) || (n_repairs && !repairs) || (cap && !out) || (data_cap && !data))
        return WMB_E_INVAL;
    *n = 0;
    size_t need = 0;
    for (size_t i = 0; i < n_lines; i++) {
        if (info[i].chain > WMB_CHAIN_S1 || line[i].len > sizeof(line[i].datagram)) return WMB_E_INVAL;
        if (info[i].crc_ok) need += line[i].len;
    }
    for (size_t i = 0; i < n_repairs; i++) {
        if (repairs[i].chain > WMB_CHAIN_S1 || repairs[i].repair.line.len > sizeof(repairs[i].repair.line.datagram)) return WMB_E_INVAL;
        if (repairs[i].repair.outcome == WMB_REP_REPAIRED) need += repairs[i].repair.line.len;
    }
    if (cap < n_lines + n_repairs || data_cap < need) return WMB_E_INVAL;
    const size_t nc_max = n_lines + n_repairs;
    if (!nc_max) return WMB_OK;
    tlg_cand *cand = (tlg_cand *)malloc(nc_max * sizeof(tlg_cand));
    tlg_rec *rec = (tlg_rec *)malloc(nc_max * sizeof(tlg_rec));
    if (!cand || !rec) { free(cand); free(rec); return WMB_E_NOMEM; }
    size_t nc = 0;
    for (size_t i = 0; i < n_lines; i++) {                      /* 1. candidates */
        tlg_cand *k = &cand[nc++];
        k->sync = info[i].sync_sample; k->d = &line[i]; k->idx = i; k->chain = info[i].chain;
        k->src = (uint8_t)(info[i].algo == WMB_ALGO_T2A ? WMB_TLG_T2A_LINE : WMB_TLG_RLA_LINE);
        k->verified = info[i].crc_ok ? 1 : 0;
    }
    for (size_t i = 0; i < n_repairs; i++) {
        const wmb_repair_record *r = &repairs[i];
        if (r->repair.outcome != WMB_REP_REPAIRED) continue;
        tlg_cand *k = &cand[nc++];
        k->sync = r->sync_sample; k->d = &r->repair.line; k->idx = n_lines + i; k->chain = r->chain;
        k->src = (uint8_t)(r->algo == WMB_ALGO_T2A ? WMB_TLG_T2A_REPAIR : WMB_TLG_RLA_REPAIR);
        k->verified = 1;
    }
    qsort(cand, nc, sizeof(tlg_cand), tlg_cand_cmp);
    size_t nr = 0;
    for (size_t g = 0; g < nc;) {                               /* 2. groups: runs of matches at most W apart */
        size_t e = g + 1;
        while (e < nc && cand[e].chain == cand[g].chain && cand[e].sync - cand[e - 1].sync <= W[cand[g].chain]) e++;
        uint32_t failed = 0;
        const size_t first = nr;
        for (size_t i = g; i < e; i++) {                        /* 3. one record per distinct verified datagram */
            if (!cand[i].verified) { failed++; continue; }
            size_t r = first;
            while (r < nr && !same_datagram(cand[i].d, rec[r].d)) r++;
            if (r == nr) {
                tlg_rec *q = &rec[nr++];
                memset(&q->t, 0, sizeof(q->t));
                q->t.decoded = 1;
                q->t.len = (uint16_t)cand[i].d->len;
                memcpy(q->t.mode, cand[i].d->mode, sizeof(q->t.mode));
                q->t.mode[2] = 0;
                q->d = cand[i].d;
                tlg_header(&q->t, q->d->datagram, q->t.len);
            }
            rec[r].t.sources |= cand[i].src;
        }
        if (nr == first) {                                      /* no verified datagram */
            tlg_rec *q = &rec[nr++];
            memset(&q->t, 0, sizeof(q->t));
            q->d = NULL;
        }
        for (size_t r = first; r < nr; r++) {
            rec[r].t.sync_sample = cand[g].sync;
            rec[r].t.chain = cand[g].chain;
            rec[r].t.failed = failed;
        }
        g = e;
    }
    qsort(rec, nr, sizeof(tlg_rec), tlg_rec_cmp);               /* 5. order */
    size_t at = 0;
    for (size_t r = 0; r < nr; r++) {
        out[r] = rec[r].t;
        if (rec[r].t.len) memcpy(data + at, rec[r].d->datagram, rec[r].t.len);
        at += rec[r].t.len;
    }
    *n = nr;
    free(cand);
    free(rec);
    return WMB_OK;
}
