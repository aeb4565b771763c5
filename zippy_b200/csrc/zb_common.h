// zb_common.h -- constants, RFC1951 tables and small helpers shared by host and device code.
//
// Everything in this header compiles both with nvcc (device + host) and with plain
// g++ (tests/test_host_units builds the Huffman / checksum maths on the CPU).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ZB_HD __host__ __device__ __forceinline__
#define ZB_HD_NOINLINE __host__ __device__ inline
#else
#define ZB_HD inline
#define ZB_HD_NOINLINE inline
#endif

// ---- geometry of the compress pipeline (see DESIGN.md "Data layout") ----
#define ZB_CHUNK_BYTES 65536      // one DEFLATE block per chunk, one CTA per chunk
#define ZB_WARPS_PER_CHUNK 8      // each warp parses one sub-chunk with a private hash table
#define ZB_SUB_BYTES (ZB_CHUNK_BYTES / ZB_WARPS_PER_CHUNK)  // 8192
#define ZB_WINDOW 32              // positions a warp examines per step (one per lane)
#define ZB_WINDOWS_PER_CHUNK (ZB_CHUNK_BYTES / ZB_WINDOW)   // 2048
#define ZB_WINDOWS_PER_SUB (ZB_SUB_BYTES / ZB_WINDOW)       // 256
#define ZB_MATCH_SLOTS 8          // a 32-byte window starts at most 8 matches (min length 4)
#define ZB_RECS_PER_SUB (ZB_SUB_BYTES / 4)    // match records a sub-chunk can hold (matches are >= 4 bytes)
#define ZB_REC_PIECE_BYTES 4096               // the records of each 4 KiB piece form one dense stream at recs[chunk][piece start / 4]
#define ZB_REC_PIECE_WINDOWS (ZB_REC_PIECE_BYTES / ZB_WINDOW)
#define ZB_RECS_PER_CHUNK (ZB_WARPS_PER_CHUNK * ZB_RECS_PER_SUB)

// ---- rsyncable compression: the content-defined chunk rule (zb_rsync.cu, DESIGN.md section 5 "Rsyncable") ----
// A format promise: members written under these values must keep their chunk starts, so they never change silently.
#define ZB_RSYNC_MIN 16384        // an accepted cut has no other candidate in the MIN bytes before it
#define ZB_RSYNC_BITS 16          // p is a candidate when the top BITS bits of its gear hash are zero
// most chunks of a member of len bytes: ceil(len / 64 KiB) + floor(len / MIN), and the one empty chunk of len 0
ZB_HD uint64_t zb_rsync_cap(uint64_t len) {
  return len == 0 ? 1 : (len + ZB_CHUNK_BYTES - 1) / ZB_CHUNK_BYTES + len / ZB_RSYNC_MIN;
}

#define ZB_NUM_LITLEN 286
#define ZB_NUM_DIST 30
#define ZB_HIST_SYMS (ZB_NUM_LITLEN + ZB_NUM_DIST)  // 316
#define ZB_HIST_WORDS (ZB_HIST_SYMS / 2)            // two u16 counters per u32 word = 158
#define ZB_MAX_MATCH 258
#define ZB_MIN_MATCH 4
#define ZB_MAX_DIST 32768

// ---- status codes (mirrors the reference's ZippyError messages; include/zippy_b200.h) ----
enum {
  ZB_OK = 0,
  ZB_ERR_INVALID_LEVEL = 1,
  ZB_ERR_INVALID_FORMAT = 2,
  ZB_ERR_UNCOMPRESS = 3,
  ZB_ERR_COMPRESS = 4,
  ZB_ERR_END_OF_BUFFER = 5,
  ZB_ERR_BYTE_BOUNDARY = 6,
  ZB_ERR_BLOCK_HEADER = 7,
  ZB_ERR_INVALID_SYMBOL = 8,
  ZB_ERR_DETECT = 9,
  ZB_ERR_METHOD = 10,
  ZB_ERR_CINFO = 11,
  ZB_ERR_HEADER = 12,
  ZB_ERR_FDICT = 13,
  ZB_ERR_CHECKSUM = 14,
  ZB_ERR_GZIP_ID = 15,
  ZB_ERR_GZIP_RESERVED = 16,
  ZB_ERR_GZIP_FLAGS = 17,
  ZB_ERR_SIZE = 18,
  ZB_ERR_DST_TOO_SMALL = 19,
  ZB_ERR_CUDA = 20,
  ZB_ERR_NOMEM = 21,
  ZB_ERR_ARG = 22,
  ZB_ERR_DICTIONARY = 23
};

enum { ZB_DF_DETECT = 0, ZB_DF_ZLIB = 1, ZB_DF_GZIP = 2, ZB_DF_DEFLATE = 3 };
// compression strategies: zlib's values (ZB200_STRATEGY_* in zippy_b200.h)
enum { ZB_STRATEGY_DEFAULT = 0, ZB_STRATEGY_FILTERED = 1, ZB_STRATEGY_HUFFMAN_ONLY = 2, ZB_STRATEGY_RLE = 3, ZB_STRATEGY_FIXED = 4 };
// the optimal parse (k_opt, the _optimal calls): a work's strategy only, never one a caller can pass
enum { ZB_STRATEGY_OPTIMAL = 5 };

// RFC 1951 section 3.2.5 tables.
#define ZB_BASE_LENGTHS                                                                          \
  { 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, \
    131, 163, 195, 227, 258 }
#define ZB_LENGTH_EXTRA \
  { 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0 }
#define ZB_BASE_DISTS                                                                         \
  { 1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, \
    2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577 }
#define ZB_DIST_EXTRA \
  { 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13 }
#define ZB_CLCL_ORDER \
  { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 }

// Distance code of a distance d in 1..32768 (RFC 1951 table, closed form).
ZB_HD int zb_dist_code(uint32_t d) {
  uint32_t v = d - 1;
  if (v < 4) return (int)v;
#if defined(__CUDA_ARCH__)
  int hb = 31 - __clz((int)v);
#else
  int hb = 31 - __builtin_clz(v);
#endif
  return 2 * hb + (int)((v >> (hb - 1)) & 1);
}
ZB_HD int zb_dist_extra_bits(int code) { return code < 4 ? 0 : (code >> 1) - 1; }
ZB_HD uint32_t zb_dist_base(int code) {
  return code < 4 ? (uint32_t)code + 1 : ((2u + (uint32_t)(code & 1)) << ((code >> 1) - 1)) + 1;
}

// Length code index (0..28) of a match length 3..258, closed form.
ZB_HD int zb_len_code(uint32_t len) {
  if (len == 258) return 28;
  uint32_t v = len - 3;
  if (v < 8) return (int)v;
#if defined(__CUDA_ARCH__)
  int hb = 31 - __clz((int)v);
#else
  int hb = 31 - __builtin_clz(v);
#endif
  return 4 * hb - 4 + (int)((v >> (hb - 2)) & 3);
}
ZB_HD int zb_len_extra_bits(int code) { return (code < 8 || code == 28) ? 0 : (code >> 2) - 1; }
ZB_HD uint32_t zb_len_base(int code) {
  if (code < 8) return (uint32_t)code + 3;
  if (code == 28) return 258;
  return ((4u + (uint32_t)(code & 3)) << ((code >> 2) - 1)) + 3;
}

// The same codes without branches (the parse converts every match with these): code and extra value of a match
// length 3..258 / a distance 1..32768.  With e = the code's extra bits, code = 4e + (v >> e) for v = len - 3 and
// 2e + (v >> e) for v = d - 1 (e = 0 covers the codes without extra bits); the extra value is v's low e bits.
ZB_HD uint32_t zb_hibit(uint32_t v) {  // index of the highest set bit of v | 1
#if defined(__CUDA_ARCH__)
  return 31u - (uint32_t)__clz((int)(v | 1u));
#else
  return 31u - (uint32_t)__builtin_clz(v | 1u);
#endif
}
ZB_HD uint32_t zb_len_code_bf(uint32_t len, uint32_t &extra) {
  const uint32_t v = len - 3u;
  const int h = (int)zb_hibit(v) - 2;
  const uint32_t e = h > 0 ? (uint32_t)h : 0u;
  const bool top = len == 258u;  // 258 has its own code, 28, with no extra bits
  extra = top ? 0u : v & ((1u << e) - 1u);
  return top ? 28u : 4u * e + (v >> e);
}
ZB_HD uint32_t zb_dist_code_bf(uint32_t d, uint32_t &extra) {
  const uint32_t v = d - 1u;
  const int h = (int)zb_hibit(v) - 1;
  const uint32_t e = h > 0 ? (uint32_t)h : 0u;
  extra = v & ((1u << e) - 1u);
  return 2u * e + (v >> e);
}

ZB_HD uint32_t zb_brev16(uint32_t v, int len) {  // reverse the low `len` bits (len<=16)
  if (len == 0) return 0u;
#if defined(__CUDA_ARCH__)
  return __brev(v) >> (32 - len);
#else
  v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
  v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
  v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
  v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
  v = (v >> 16) | (v << 16);
  return v >> (32 - len);
#endif
}
