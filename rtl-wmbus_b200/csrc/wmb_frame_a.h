/*
 * wmb_frame_a.h -- the CRC block layout of frame format A (t1_c1_packet_decoder.h:471-506, CRC strip :551-592), shared
 * by the device repair K4R (wmb_kernels.cuh) and its host twin wmb_frame_repair() (wmb_framer.c), so that the two cannot
 * drift apart.  A telegram of len >= 12 bytes has a 12-byte first block and 18-byte blocks after it, the last one
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

#endif
