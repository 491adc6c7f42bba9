/*
 * wmb_frame_a.h -- the CRC block layout of frame format A (t1_c1_packet_decoder.h:471-506, CRC strip :551-592), shared
 * by the device repair K4R (wmb_kernels.cuh) and its host twin wmb_frame_repair() (wmb_framer.c), so that the two cannot
 * drift apart (and, below, the T1 soft repair's symbol scoring and the S1 soft repair's pair scoring, for K4S and
 * wmb_frame_repair_t1_soft() / wmb_frame_repair_s1_soft()).  A telegram
 * of len >= 12 bytes has a 12-byte first block and 18-byte blocks after it, the last one
 * shorter; each block ends in its two CRC bytes.
 */
#ifndef WMB_FRAME_A_H
#define WMB_FRAME_A_H

#include <stdint.h>

#ifdef __CUDACC__
#define WMB_FA static inline __host__ __device__
#else
#define WMB_FA static inline
#endif

WMB_FA uint32_t wmb_nblk_a(uint32_t len) { return 1 + (len - 12 + 17) / 18; }

WMB_FA uint32_t wmb_blk_off_a(uint32_t j) { return j ? 12 + 18 * (j - 1) : 0; }

WMB_FA uint32_t wmb_blk_len_a(uint32_t len, uint32_t j)
{
    const uint32_t off = wmb_blk_off_a(j);
    return j ? ((len - off >= 18) ? 18 : len - off) : 12;
}

/* byte i of the CRC-stripped datagram is this byte of the telegram */
WMB_FA uint32_t wmb_strip_src_a(uint32_t i) { return i < 10 ? i : 12 + 18 * ((i - 10) / 16) + (i - 10) % 16; }

/* Frame format B (t1_c1_packet_decoder.h:508-536, CRC strip :595-636): 128-byte blocks from byte 0, the last one shorter,
 * each ending in its two CRC bytes.  Shared by the C1 soft repair K4S and its host twin wmb_frame_repair_soft(). */
WMB_FA uint32_t wmb_nblk_b(uint32_t len) { return (len + 127) / 128; }

WMB_FA uint32_t wmb_blk_off_b(uint32_t j) { return 128 * j; }

WMB_FA uint32_t wmb_blk_len_b(uint32_t len, uint32_t j) { return (len - 128 * j >= 128) ? 128 : len - 128 * j; }

/* byte i of the CRC-stripped datagram is this byte of the telegram (the strip then lowers byte 0 by 2 per block) */
WMB_FA uint32_t wmb_strip_src_b(uint32_t i) { return 128 * (i / 126) + i % 126; }

/* T1 soft repair (wmbus_b200_framer.h), shared by K4S and its host twin wmb_frame_repair_t1_soft(): the 3-out-of-6 code
 * word of nibble n (t1_c1_packet_decoder.h:50-65), and the ML value, runner-up and delta of one symbol from its six
 * centred chip values y[0..6), first chip first.  C(w) = 2 sum of y over w's 1-chips - sum of y, so comparing the first
 * term is enough; ties go to the lower nibble. */
WMB_FA uint32_t wmb_enc3of6(uint32_t n)
{
    return (uint32_t)(((n < 8 ? 0x131A191C0B0E0D16ull : 0x293231342326252Cull) >> (8 * (n & 7u))) & 0xFFu);
}

WMB_FA void wmb_t1_sym_ml(const int64_t *y, uint32_t *ml, uint32_t *ru, int64_t *delta)
{
    int64_t best = 0, second = 0;
    uint32_t b = 16, s = 16;
    for (uint32_t n = 0; n < 16; n++) {
        const uint32_t w = wmb_enc3of6(n);
        int64_t c = 0;
        for (uint32_t j = 0; j < 6; j++) if (w >> (5 - j) & 1u) c += y[j];
        if (b == 16 || c > best) { s = b; second = best; b = n; best = c; }
        else if (s == 16 || c > second) { s = n; second = c; }
    }
    *ml = b; *ru = s; *delta = 2 * (best - second);
}

/* S1 soft repair (wmbus_b200_framer.h), shared by K4S and its host twin wmb_frame_repair_s1_soft(): Manchester pair p
 * from its chips' soft values v1, v2 (-32768: none) and hard chips a, c.  *ml is its ML bit; the result its search key
 * (has a value, |d|, p) as one integer, has << 29 | |d| << 12 | p: |d| <= 65534 < 2^17, p < 8 * 296 < 2^12. */
WMB_FA uint32_t wmb_s1_pair(int32_t v1, int32_t v2, uint32_t a, uint32_t c, uint32_t p, uint32_t *ml)
{
    const int none = v1 == -32768 || v2 == -32768;
    const int32_t d = none ? 0 : v2 - v1;
    *ml = d > 0 ? 1u : d < 0 ? 0u : (a != c ? c : 0u);
    return (none ? 0u : 1u << 29) | (uint32_t)(d < 0 ? -d : d) << 12 | p;
}

#endif
