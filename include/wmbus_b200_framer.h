/*
 * wmbus_b200_framer.h -- the host-side framers of libwmbus_b200.so as a C ABI of their own.
 *
 * Frame-at-once replacements for the reference's per-bit decoder state machines
 * t1_c1_packet_decoder() (t1_c1_packet_decoder.h:649-712) and s1_packet_decoder()
 * (s1_packet_decoder.h:233-282): a candidate frame (the bit carrying the access-code flag plus
 * the bits that follow it, as wmb_poll() hands them out) is decoded in one pass -- 3-out-of-6 /
 * NRZ / Manchester, L-field, RSSI abort, block CRCs, CRC strip -- and formatted as the
 * reference prints it (t1_c1_packet_decoder.h:670-699, rtl_wmbus_util.h:10-39).
 *
 * wmb_decode_frames() (wmbus_b200.h) is these functions plus the stream-order bookkeeping; a
 * caller who keeps its own bookkeeping (or only wants the CRC / line format) binds them directly.
 * The default path decodes on the device (kernel K4); wmb_frame_decode() is its host twin and
 * wmb_frame_decode_device() lets a test compare the two candidate by candidate.  wmb_frame_repair() repairs T1 / S1
 * candidates that lost a few chips (erasure decoding checked by the block CRCs), with the device twin
 * wmb_frame_repair_device(); wmb_frame_repair_soft() / wmb_frame_repair_soft_device() also repair C1 candidates from the
 * soft values of their bits (wmb_set_soft_bits, wmb_frame_soft), and wmb_frame_repair_t1_soft() /
 * wmb_frame_repair_t1_soft_device() the T1 candidates that erasure repair gives up on, and wmb_frame_repair_s1_soft() /
 * wmb_frame_repair_s1_soft_device() the S1 ones, from the soft values of their chips (wmb_set_soft_bits_s1).
 */
#ifndef WMBUS_B200_FRAMER_H
#define WMBUS_B200_FRAMER_H

#include <stddef.h>
#include <stdint.h>
#include "wmbus_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { WMB_DEC_ABORT = 0, WMB_DEC_LINE = 1, WMB_DEC_NEED_MORE = 2 };

typedef struct wmb_decoded {
    int      status;            /* WMB_DEC_*                                            */
    uint32_t consumed;          /* bits consumed incl. the flagged one (>= 1)           */
    uint64_t end_sample;        /* decimated sample of the last consumed bit            */
    char     mode[3];           /* "T1" / "C1" / "S1"                                   */
    uint8_t  crc_ok, ok_3of6;
    uint32_t packet_rssi, current_rssi;
    uint32_t serial;            /* LINK_LAYER_IDENT_NO                                  */
    uint32_t len;               /* datagram bytes after the CRC strip                   */
    uint8_t  datagram[292];
} wmb_decoded;

/* Decode one candidate on the host (t1_c1_packet_decoder.h:272-460, s1_packet_decoder.h:132-282).
 * WMB_DEC_NEED_MORE is returned when the bit list ends while the framer is still receiving. */
void wmb_frame_decode(const wmb_frame *f, wmb_decoded *out);

/* The same decode done by the device framer (kernel K4), n frames at once. */
int wmb_frame_decode_device(wmb_ctx *ctx, const wmb_frame *frames, size_t n, wmb_decoded *out);

/* ---- erasure repair of one candidate ----------------------------------------------------------------------------
 * T1 (3-out-of-6) and S1 (Manchester) say where a chip went wrong: one flipped chip makes a 6-bit word that is no
 * code word (weight 2 or 4), or a "00" / "11" chip pair.  The block CRCs then tell which filling of those erasures
 * is right.  With e_max in 1..3:
 *   1. Candidates: a frame whose decode (wmb_frame_decode) is a line with crc_ok = 0, and an S1 frame whose decode
 *      aborts on a Manchester violation after the L-field byte.  The L-field is never repaired.  The bit list must reach
 *      P = 1 + 12 len (T1) or 1 + 16 len (S1) bits (else TRUNCATED) and no bit before bit P - 1 may have rssi < 5 (else
 *      UNREPAIRABLE: the RSSI abort stays an abort).  C1 is NRZ and has no erasures.
 *   2. Erasures: a T1 data or CRC symbol that is no code word.  Weight 2 or 4: its fillings are the code words at
 *      Hamming distance 1 (2 to 4 of them); weight 0, 1, 5, 6 and the invalid weight-3 words 7, 21, 42, 56 make the
 *      frame UNREPAIRABLE.  An S1 "00" / "11" pair: fillings 0 and 1.
 *   3. Blocks of frame format A (12 bytes, then 18): a block with more than e_max erasures makes the frame TOO_MANY.
 *      Otherwise, in block order, a block must have exactly one filling (of at most 4^e or 2^e) that passes its CRC --
 *      as received when it has no erasure.  The first block with none makes the frame UNREPAIRABLE, with two or more
 *      AMBIGUOUS.
 *   4. REPAIRED: every block passes and at least one erasure was filled.  `line` is then the line the reference would
 *      print for the repaired bytes: crc_ok = ok_3of6 = 1, CRC-stripped datagram, consumed = P, end_sample = the
 *      sample of bit P - 1, packet_rssi / current_rssi at bits 1 and P - 1.
 * Why wrong repairs stay rare: DESIGN.md section 8. */
enum { WMB_REP_NONE = 0,          /* not a candidate (a good line, another abort, repair off)                    */
       WMB_REP_REPAIRED = 1, WMB_REP_AMBIGUOUS = 2, WMB_REP_TOO_MANY = 3, WMB_REP_UNREPAIRABLE = 4,
       WMB_REP_TRUNCATED = 5 };

typedef struct wmb_repaired {
    int         outcome;        /* WMB_REP_*                                            */
    uint32_t    erasures;       /* REPAIRED: erasures filled                            */
    uint32_t    blocks;         /* REPAIRED: blocks that had erasures                   */
    uint32_t    had_line;       /* 1: the decode was a line with crc_ok = 0; 0: an S1 abort */
    wmb_decoded line;           /* REPAIRED: the repaired line (status WMB_DEC_LINE)    */
} wmb_repaired;

/* Repair one candidate on the host, e_max = 0 (nothing is repaired: WMB_REP_NONE) .. 3; else WMB_E_INVAL. */
int wmb_frame_repair(const wmb_frame *f, uint32_t e_max, wmb_repaired *out);

/* The same repair done on the device (kernel K4R behind K4), n frames at once. */
int wmb_frame_repair_device(wmb_ctx *ctx, const wmb_frame *frames, size_t n, uint32_t e_max, wmb_repaired *out);

/* ---- erasure repair on the streaming path (wmb_push / wmb_push_device / wmb_process*) ------------------------------
 * Off by default.  wmb_set_repair(ctx, e_max), e_max 1..3, turns it on (0: off); e_max > 3 is WMB_E_INVAL, and so is a
 * manual_frames context (it repairs its polled frames with wmb_frame_repair_device).  Like wmb_set_line_quality it is
 * valid before the first push or right after wmb_reset / wmb_seek (else WMB_E_STATE) and survives both.
 *   1. Candidates: exactly the frames that the context's own framer books -- the stream-order rule accepted them (a
 *      match that lies inside a telegram already accepted on its stream is ignored) and the match lies in the line
 *      window (wmb_set_line_window) -- whose decode is a candidate of wmb_frame_repair above: a line with crc_ok = 0, or
 *      an S1 abort on a Manchester violation after the L-field.
 *   2. Each is repaired as wmb_frame_repair defines, on its bit list once that holds P bits.  No record is made when the
 *      list ends before P (a run-length reset, the end of input) or when the outcome is NONE: every record is REPAIRED,
 *      AMBIGUOUS, TOO_MANY or UNREPAIRABLE.  (A REPAIRED one whose datagram found no room in the batch's pool is not
 *      reported either; the batch counts as an overflow batch.)
 *   3. Records come out in (end_sample, chain * 2 + (algo == t2a), sync_sample) order; end_sample is the sample of bit
 *      P - 1 (of a C1 line, which is never repaired, its last bit), and a record becomes final in the gather whose batch
 *      produced that bit.
 *   4. A repair is an additional report: the lines and their info / quality records, the bursts, the band survey, the
 *      busy bookkeeping and every wmb_stats field but kernel_launches (one more per gather) and d2h_bytes stay as they
 *      are with repair off. */
typedef struct wmb_repair_record {
    uint64_t     sync_sample;   /* access-code match (decimated sample)                 */
    uint64_t     end_sample;    /* decimated sample of bit P - 1 (a C1 line: its last bit) */
    uint8_t      chain, algo;   /* WMB_CHAIN_*, WMB_ALGO_*                              */
    uint8_t      soft_t1;       /* 1: the T1 soft rule (wmb_set_repair_t1_soft) decided this record */
    uint8_t      soft_s1;       /* 1: the S1 soft rule (wmb_set_repair_s1_soft) decided this record */
    uint8_t      reserved[4];
    wmb_repaired repair;        /* outcome; REPAIRED: the repaired line                 */
} wmb_repair_record;

int wmb_set_repair(wmb_ctx *ctx, uint32_t e_max);

/* Hand out at most cap of the queued records, in order; the rest stay queued.  *n: records written. */
int wmb_take_repairs(wmb_ctx *ctx, wmb_repair_record *out, size_t cap, size_t *n);

/* ---- soft values of the T1/C1 chain's bits ------------------------------------------------------------------------
 * How sure the slicer was of a bit.  Bit event e of a T1/C1 stream lies at decimated sample m.  Its chip centre is
 *   t2a:  c = m - WMB_SOFT_D_T2;
 *   rla:  c = m - WMB_SOFT_D_RL - 8 (n - 1 - i), e being the i-th of the n events that share sample m (one edge emits
 *         its whole run of bits at one sample).
 * v = clamp(floor(sum over q in [c - 2, c + 3) of rint(dphi[q] * 2^24) / 2^12), -32767, 32767), as an int16, where dphi
 * is the post-FIR discriminator output before the DC block (the signal the carrier-offset and quality windows read).
 * WMB_SOFT_NONE means "no value": the window starts before the first sample pushed since the last reset / seek, or
 * n - 1 - i > 63.  The values are sums of exact integer terms: they do not depend on batch cuts or thread order.
 * D_RL maximises the mean of (2 bit - 1) v over clean C1 telegrams.  D_T2 does so only among the values >= 2, for which
 * the window ends at the event's own sample: a deliberate departure from the plain argmax (D = 1, 4 % more mean margin),
 * whose window would need the sample after the event, which the event's batch may not hold (DESIGN.md section 8).
 * wmb_set_soft_bits(ctx, on) makes the device gather of a manual_frames context compute them (WMB_E_INVAL on any other
 * context: its soft values serve wmb_set_repair_soft below); the setter follows wmb_set_line_quality's state rules and
 * the setting survives wmb_reset / wmb_seek.  wmb_frame_soft() returns them for a frame of the last wmb_poll: parallel to
 * f->bits, valid as long as f->bits; NULL for S1 frames (unless wmb_set_soft_bits_s1 is on) or when soft values are off. */
#define WMB_SOFT_NONE  (-32768)
#define WMB_SOFT_D_T2  2
#define WMB_SOFT_D_RL  7

int wmb_set_soft_bits(wmb_ctx *ctx, int on);
int wmb_frame_soft(wmb_ctx *ctx, const wmb_frame *f, const int16_t **soft);

/* ---- C1 soft repair of one candidate --------------------------------------------------------------------------------
 * C1 is NRZ: a wrong bit leaves no trace in the code, only in its soft value.  With k_max in 1..WMB_SOFT_K_MAX:
 *   1. Candidates: a C1 frame (format A or B) whose decode is a line with crc_ok = 0 and len >= 12 bytes (else
 *      UNREPAIRABLE).  P = 17 + 8 len; byte l occupies frame bits [17 + 8 l, 25 + 8 l).  The L byte is never flipped.
 *   2. Reliability: over the bits [17, P) without WMB_SOFT_NONE, n1 and S1 are the count and the sum of v of the bits
 *      decided 1, n0 and S0 those of the bits decided 0.  r_j = (2 bit_j - 1) (v_j 2 n0 n1 - (S1 n0 + S0 n1)) in int64,
 *      the distance from a threshold midway between the telegram's own tone means; if n0 n1 = 0, r_j = (2 bit_j - 1) v_j.
 *      A bit without a value ranks lowest.
 *   3. Blocks: frame A as wmb_frame_repair (12 bytes, then 18); frame B 128-byte blocks from byte 0.  A block that
 *      passes its CRC as received is left alone.
 *   4. Search: in a failing block take the K = min(k_max, flippable bits) bits of lowest r (ties: lower bit index).
 *      Exactly one of the 2^K - 1 non-zero flip patterns must pass the block's CRC.  In block order, the first block
 *      where none does makes the frame UNREPAIRABLE, where two or more do AMBIGUOUS.
 *   5. REPAIRED: every block passes.  `line` is the line the reference would print for the corrected bytes (crc_ok =
 *      ok_3of6 = 1, CRC-stripped datagram, consumed = P, end_sample = bit P - 1); erasures = bits flipped, blocks = blocks
 *      changed, had_line = 1.
 * Any other frame, or k_max = 0, or soft = NULL, is repaired exactly as wmb_frame_repair(f, e_max) does.
 * Why a wrong repair stays rare: DESIGN.md section 8. */
#define WMB_SOFT_K_MAX 6

int wmb_frame_repair_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t k_max, wmb_repaired *out);

/* The same done on the device (K4, the erasure repair K4R, then the soft repair K4S), n frames at once; softs[i] is
 * frame i's soft values (NULL: none). */
int wmb_frame_repair_soft_device(wmb_ctx *ctx, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                 uint32_t e_max, uint32_t k_max, wmb_repaired *out);

/* C1 soft repair on the streaming path.  wmb_set_repair_soft(ctx, k_max), k_max 0 (off, the default) .. WMB_SOFT_K_MAX,
 * else WMB_E_INVAL; WMB_E_INVAL on a manual_frames context; the state rules of wmb_set_repair, and the setting survives
 * wmb_reset / wmb_seek.  While wmb_set_repair has repair on, the C1 candidates of the streaming repair (lines with
 * crc_ok = 0) follow the rule above (wmb_frame_repair_soft with the soft values the gather computes) instead of being
 * UNREPAIRABLE; their record's end_sample is bit P - 1, the line's last bit, as before.  T1 and S1 candidates are
 * unchanged.  wmb_boundary_state appends k_max when it is not 0. */
int wmb_set_repair_soft(wmb_ctx *ctx, uint32_t k_max);

/* ---- T1 soft repair of one candidate --------------------------------------------------------------------------------
 * The erasure rule gives up on a T1 block with more than e_max invalid symbols, on a symbol with no code word at distance
 * 1, and on two wrong chips that made another valid code word.  The soft values decide all three.  T1 frame layout (as
 * K4 reads it): bit 0 the flagged bit, byte l at bits [1 + 12 l, 13 + 12 l), its high-nibble symbol first, a symbol's
 * first chip the MSB of its 6-bit word; len = wmb_tlg_len_a(L), P = 1 + 12 len; frame format A.  With s_max in
 * 1..WMB_SOFT_K_MAX:
 *   1. Candidates: a T1 frame whose decode is a line with crc_ok = 0 and len >= 12, whose bit list reaches P, with no bit
 *      before P - 1 of rssi < 5 (a line implies both), with soft values, and for which wmb_frame_repair(f, e_max) ends
 *      in TOO_MANY or UNREPAIRABLE.  The erasure rule runs first and its REPAIRED, AMBIGUOUS, TRUNCATED and NONE stand,
 *      so the repairs with this rule on are a superset of those without it.  The L byte (bits [1, 13)) never changes.
 *   2. Centring: over the chips [13, P) with a value, n1 and S1 are the count and the sum of v of the chips decided 1,
 *      n0 and S0 those of the chips decided 0.  y_j = v_j 2 n0 n1 - (S1 n0 + S0 n1) in int64 (K4S's C1 centring); if
 *      n0 n1 = 0, y_j = v_j; a chip without a value has y_j = 0.
 *   3. Symbols: code word w (one of the 16) scores C(w) = sum over the symbol's six chips of (2 w_j - 1) y_j.  ML is
 *      the argmax of C (ties: the lower nibble), the runner-up the argmax over the other 15 (same ties), and
 *      delta = C(ML) - C(runner-up) >= 0.  A symbol with a chip without a value ranks before every symbol without one.
 *   4. Blocks: frame A's (12 bytes, then 18).  A block that passes as received (every symbol valid, CRC passes) is left
 *      alone.  In a failing block every searchable symbol takes its ML value and the K = min(s_max, searchable symbols)
 *      of lowest delta (ties: lower symbol index) are searched; the first block's searchable symbols are those of bytes
 *      1..11.  Exactly one of the 2^K patterns must pass the block's CRC: pattern 0 is pure ML, set bit u replaces
 *      searched symbol u's ML value by its runner-up.  In block order, the first block where none does makes the frame
 *      UNREPAIRABLE, where two or more do AMBIGUOUS.
 *   5. REPAIRED: every block passes.  `line` is the line the reference would print for the corrected bytes (crc_ok =
 *      ok_3of6 = 1, CRC-stripped datagram, consumed = P, end_sample = bit P - 1, packet_rssi / current_rssi at bits 1 and
 *      P - 1); erasures = the symbols whose nibble differs from the hard decode (an invalid symbol differs; at most
 *      255 are counted), blocks = the blocks changed, had_line = 1.
 * When the rule ran, its outcome replaces the erasure rule's.  Any other frame, s_max = 0 or soft = NULL is repaired
 * exactly as wmb_frame_repair(f, e_max) does.  All magnitudes fit int64: |y| < 2^39, |C| < 2^42.  Why a wrong repair
 * stays rare: DESIGN.md section 8. */
int wmb_frame_repair_t1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out);

/* The same done on the device (K4, the erasure repair K4R, then K4S with k_max = 0), n frames at once; softs[i] is frame
 * i's soft values (NULL: none). */
int wmb_frame_repair_t1_soft_device(wmb_ctx *ctx, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                    uint32_t e_max, uint32_t s_max, wmb_repaired *out);

/* T1 soft repair on the streaming path.  wmb_set_repair_t1_soft(ctx, s_max), s_max 0 (off, the default) ..
 * WMB_SOFT_K_MAX, else WMB_E_INVAL; WMB_E_INVAL on a manual_frames context; the state rules of wmb_set_repair_soft, the
 * setting survives wmb_reset / wmb_seek and is independent of it.  While wmb_set_repair has repair on, the T1 candidates
 * of the streaming repair follow the rule above with the soft values the gather computes; a record the rule decided has
 * soft_t1 = 1.  Records become final at bit P - 1, as before.  wmb_boundary_state appends s_max when it is not 0. */
int wmb_set_repair_t1_soft(wmb_ctx *ctx, uint32_t s_max);

/* ---- soft values of the S1 chain's chips --------------------------------------------------------------------------
 * How sure the slicer was of an S1 chip.  Bit event e of an S1 stream lies at decimated sample m.  Its chip centre is
 *   t2a:  c = m - WMB_SOFT_S1_D_T2;
 *   rla:  c = m - WMB_SOFT_S1_D_RL - 24 (n - 1 - i), e being the i-th of the n events that share sample m.  24 is the
 *         nominal samples per chip (runlength_algorithm_reset_s1); a valid Manchester run is at most 2 chips long, so
 *         the nominal spacing is off by less than a sample.
 * v = clamp(floor(sum over q in [c - 8, c + 8) of rint(dphi[q] * 2^24) / 2^WMB_SOFT_S1_SHIFT), -32767, 32767), as an
 * int16, over the same post-FIR, pre-DC-block dphi as the T1/C1 values.  WMB_SOFT_NONE: the window starts before the
 * first sample pushed since the last reset / seek, or n - 1 - i > 31 (so the window stays inside the dphi history).
 * Both windows end at or before the event's own sample, which the event's batch holds: the delays are >= 7.  The delays
 * maximise the mean of (2 chip - 1) v over clean S1 telegrams (DESIGN.md section 8).
 * wmb_set_soft_bits_s1(ctx, on) makes the device gather of a manual_frames context compute them (WMB_E_INVAL on any
 * other context: its S1 values serve wmb_set_repair_s1_soft below), with wmb_set_soft_bits' state rules; the setting
 * survives wmb_reset / wmb_seek and is independent of wmb_set_soft_bits.  With it on, wmb_frame_soft() returns the values
 * of S1 frames; with it off (the default) it returns NULL for them. */
#define WMB_SOFT_S1_D_T2   7
#define WMB_SOFT_S1_D_RL   13
#define WMB_SOFT_S1_SHIFT  14

int wmb_set_soft_bits_s1(wmb_ctx *ctx, int on);

/* ---- S1 soft repair of one candidate --------------------------------------------------------------------------------
 * Manchester sends every bit as one chip on each tone, so d = v(second chip) - v(first chip) decides a bit without an
 * estimate of the tone means.  S1 frame layout (as K4 reads it): bit 0 the flagged bit, byte l at bits
 * [1 + 16 l, 17 + 16 l), data bit b of the byte (MSB first) the pair (1 + 16 l + 2 b, 2 + 16 l + 2 b): "01" = 1,
 * "10" = 0; pair index 8 l + b; len = wmb_tlg_len_a(L), P = 1 + 16 len; frame format A.  With s_max in
 * 1..WMB_SOFT_K_MAX:
 *   1. Candidates: an S1 frame whose decode is a line with crc_ok = 0 or an abort on a Manchester violation after the L
 *      byte, with len >= 12, whose bit list reaches P, with no bit before P - 1 of rssi < 5 (an RSSI abort stays one),
 *      with soft values, and for which wmb_frame_repair(f, e_max) ends in TOO_MANY or UNREPAIRABLE.  Its REPAIRED,
 *      AMBIGUOUS, TRUNCATED and NONE stand, so the repairs with this rule on are a superset of those without it.  The L
 *      byte never changes.
 *   2. Pairs: d = v2 - v1 in int32 (v1 the first chip's value); a pair with a chip without a value has d = 0 and ranks
 *      before every pair with values.  The ML bit is 1 if d > 0, 0 if d < 0, and if d = 0 the received bit when the pair
 *      is valid, else 0.  Its reliability is |d|.
 *   3. Blocks: frame A's (12 bytes, then 18).  A block without a violation that passes its CRC as received is left
 *      alone.  In a failing block every searchable pair (all of the block's, but the L byte's in the first block) takes
 *      its ML bit, and the K = min(s_max, searchable pairs) of lowest key (has a value, |d|, pair index) are searched.
 *      Exactly one of the 2^K patterns must pass the block's CRC: pattern 0 is pure ML, set bit u flips searched pair
 *      u.  In block order, the first block where none does makes the frame UNREPAIRABLE, where two or more do
 *      AMBIGUOUS.
 *   4. REPAIRED: every block passes.  `line` is the line the reference would print for the corrected bytes (crc_ok =
 *      ok_3of6 = 1, CRC-stripped datagram, consumed = P, end_sample = bit P - 1, packet_rssi / current_rssi at bits 1 and
 *      P - 1); erasures = the bits that differ from the hard decode (a violation differs; at most 255 are counted),
 *      blocks = the blocks changed, had_line = 1 for a line and 0 for an abort.
 * When the rule ran, its outcome replaces the erasure rule's.  Any other frame, s_max = 0 or soft = NULL is repaired
 * exactly as wmb_frame_repair(f, e_max) does.  Why a wrong repair stays rare: DESIGN.md section 8. */
int wmb_frame_repair_s1_soft(const wmb_frame *f, const int16_t *soft, uint32_t e_max, uint32_t s_max, wmb_repaired *out);

/* The same done on the device (K4, the erasure repair K4R, then K4S), n frames at once; softs[i] is frame i's soft values
 * (NULL: none). */
int wmb_frame_repair_s1_soft_device(wmb_ctx *ctx, const wmb_frame *frames, const int16_t *const *softs, size_t n,
                                    uint32_t e_max, uint32_t s_max, wmb_repaired *out);

/* S1 soft repair on the streaming path.  wmb_set_repair_s1_soft(ctx, s_max), s_max 0 (off, the default) ..
 * WMB_SOFT_K_MAX, else WMB_E_INVAL; WMB_E_INVAL on a manual_frames context; the state rules of wmb_set_repair_t1_soft,
 * the setting survives wmb_reset / wmb_seek and is independent of the C1 and T1 settings.  While wmb_set_repair has
 * repair on, the S1 candidates of the streaming repair follow the rule above with the soft values the gather computes; a
 * record the rule decided has soft_s1 = 1.  Records become final at bit P - 1, as before.  wmb_boundary_state appends a
 * tag and s_max when s_max is not 0. */
int wmb_set_repair_s1_soft(wmb_ctx *ctx, uint32_t s_max);

/* ---- telegrams: one record per transmission, from both bit syncs and the repairs ----------------------------------
 * Each chain runs two bit syncs, so one transmission usually gives two lines (t2a and rla), and with repair on a
 * REPAIRED record beside a CRC-failed twin.  wmb_group_telegrams() joins them by this rule:
 *   1. Candidates, per chain: every line (CRC ok or not) and every repair record whose outcome is WMB_REP_REPAIRED.
 *      A candidate is verified when it is a CRC-ok line or a repaired line; its datagram is then the datagram column
 *      (CRC bytes removed: wmb_decoded.datagram[0 .. len)).
 *   2. Same transmission: two candidates of one chain whose access-code matches (sync_sample) lie at most W[chain]
 *      decimated samples apart belong together; a group is the transitive closure.  Spans are not compared: the
 *      end_sample of a failed candidate comes from an L-field that may itself be wrong.  W is WMB_TLG_W_T1C1 /
 *      WMB_TLG_W_S1, chosen from the distance of the t2a and rla matches of one telegram (DESIGN.md section 8).
 *   3. Records: one per distinct verified datagram of a group (the same mode and the same bytes), decoded = 1, with
 *      sources the WMB_TLG_* bits of the candidates that carry it.  failed counts the group's candidates that are not
 *      verified (a CRC-failed line, also when its repair is in the group).  A group without a verified candidate gives
 *      one record with decoded = 0, its failed count, no bytes and no valid header field.
 *   4. Header fields, from the datagram (L C M M A A A A V T CI ...): l = byte 0, c = byte 1, m = bytes 2..3 (little
 *      endian) and manuf its three letters ((m >> 10) & 31) + 64, ((m >> 5) & 31) + 64, (m & 31) + 64, id = bytes 4..7
 *      (little endian: the line's LINK_LAYER_IDENT_NO column), version = byte 8, type = byte 9, ci = byte 10.  valid
 *      holds the WMB_TLG_F_* bit of each field the datagram is long enough for; the others are 0.
 *   5. Order: sync_sample is the group's earliest match (all records of a group share it); records are ordered by
 *      (sync_sample, chain), the records of one group by (mode, len, bytes). */
#define WMB_TLG_W_T1C1 128
#define WMB_TLG_W_S1   256

#define WMB_TLG_T2A_LINE   1u
#define WMB_TLG_RLA_LINE   2u
#define WMB_TLG_T2A_REPAIR 4u
#define WMB_TLG_RLA_REPAIR 8u

#define WMB_TLG_F_L       1u
#define WMB_TLG_F_C       2u
#define WMB_TLG_F_M       4u
#define WMB_TLG_F_ID      8u
#define WMB_TLG_F_VERSION 16u
#define WMB_TLG_F_TYPE    32u
#define WMB_TLG_F_CI      64u

typedef struct wmb_telegram {
    uint64_t sync_sample;     /* the group's earliest access-code match (decimated sample)                      */
    uint32_t id;              /* bytes 4..7, little endian                                                      */
    uint16_t m;               /* bytes 2..3, little endian                                                      */
    uint16_t len;             /* datagram bytes (0 when decoded = 0)                                            */
    uint32_t failed;          /* the group's candidates without a verified datagram                            */
    uint8_t  chain;           /* WMB_CHAIN_*                                                                    */
    uint8_t  decoded;
    uint8_t  sources;         /* WMB_TLG_* bits                                                                 */
    uint8_t  valid;           /* WMB_TLG_F_* bits                                                               */
    char     mode[3];         /* "T1", "C1", "S1"; "" when decoded = 0                                          */
    char     manuf[4];        /* three letters; "" without WMB_TLG_F_M                                          */
    uint8_t  l, c, version, type, ci;
    uint8_t  pad[4];
} wmb_telegram;

/* The rule above over n_lines lines (info[i] and their decodes line[i]: sync_sample, chain, algo and crc_ok of info,
 * mode, len and datagram of line) and n_repairs repair records (those not REPAIRED are ignored), in any order.  The
 * records go to out in order and their datagrams, concatenated, to data.  out must hold n_lines + n_repairs records and
 * data_cap the sum of len over the verified candidates (bounds that hold for any input), else WMB_E_INVAL.  *n receives
 * the number of records. */
int wmb_group_telegrams(const wmb_line_info *info, const wmb_decoded *line, size_t n_lines,
                        const wmb_repair_record *repairs, size_t n_repairs,
                        wmb_telegram *out, size_t cap, uint8_t *data, size_t data_cap, size_t *n);

/* Telegrams on the streaming path.  wmb_set_telegrams(ctx, on), on 0 (off, the default) or 1; WMB_E_INVAL on a
 * manual_frames context (its caller frames its own candidates: it calls wmb_group_telegrams); the state rules of
 * wmb_set_repair, and the setting survives wmb_reset / wmb_seek.  On, the context keeps its lines and (repair on) its
 * REPAIRED records and groups them as wmb_group_telegrams does.  A group is handed out once it is final: no telegram of
 * its chain still in flight (wmb_pending_before's condition) and no match still to come lies within W of a member, so
 * neither a line nor a repair can join it later; and once no group still to come can come before it.  After the end of
 * input (flush) every group is final.  The records do not depend on batch size, push size or thread order.  Off, the
 * context keeps nothing.  It is host work only: no launch and no copy. */
int wmb_set_telegrams(wmb_ctx *ctx, int on);

/* Copy whole records in order: recs[i] and its len bytes, concatenated in data.  Stops at cap records or when the next
 * record's bytes do not fit data_cap; *n receives the number copied.  Records not taken stay queued. */
int wmb_take_telegrams(wmb_ctx *ctx, wmb_telegram *recs, size_t cap, uint8_t *data, size_t data_cap, size_t *n);

/* CRC-16, polynomial 0x3D65, complemented (t1_c1_packet_decoder.h:463-469) */
uint16_t wmb_crc16(const uint8_t *data, size_t n);

/* "MODE;CRC_OK;3OUTOF6OK;TIMESTAMP;PACKET_RSSI;CURRENT_RSSI;IDENT;0xHEX\n"
 * (t1_c1_packet_decoder.h:670-699); returns the length written (excluding NUL). */
size_t wmb_format_line(const wmb_decoded *d, const char *algo_prefix, const char *timestamp,
                       char *buf, size_t cap);

/* YYYY-MM-DD HH:MM:SS.uuuuuu local time (rtl_wmbus_util.h:10-39) */
void wmb_make_time_string(char *ts, size_t n);

#ifdef __cplusplus
}
#endif
#endif
