// zb_kernels.h -- launch interface between the C-ABI layer (zb_api.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "zb_common.h"
#include "zb_crc.h"
#include "zb_huff.h"

// One unit of compress work: <= 64 KiB of one member, one DEFLATE block.
struct ZbChunkDesc {
  uint64_t src_off;   // byte offset of the chunk in the source buffer
  uint32_t len;       // 0..65536
  uint32_t member;    // index of the input this chunk belongs to
  uint32_t flags;     // ZB_CHUNK_*
  uint32_t pad;       // k_lz2: bytes of the member's preceding data staged as history (<= 32768)
};
#define ZB_CHUNK_FIRST 1u  // first chunk of its member in this launch group: places member_off
#define ZB_CHUNK_LAST 2u   // last chunk of its member: BFINAL, then the trailer
#define ZB_CHUNK_HEAD 4u   // the member's gzip / zlib header goes in front of this chunk (a stream's later
                           // launches continue a member whose header an earlier launch wrote: FIRST without HEAD)
#define ZB_CHUNK_DICT 8u   // k_lz2: the chunk's `pad` bytes of history are the end of the dictionary window, not src

// The part of a member compressed before this launch (a compress stream): raw CRC-32 and Adler-32 of its
// bytes and their count.  The empty prefix is {0, 1, 0}.
struct ZbMemberCarry {
  uint32_t crc_raw;
  uint32_t adler;
  uint64_t bytes;
};

struct ZbChunkCheck {
  uint32_t crc_raw;   // init-0 CRC of the chunk bytes
  uint32_t adler;     // Adler-32 of the chunk bytes as a standalone message
};

// One member's preset dictionary D.  wend: just past the window W (the last win_len = min(32768, |D|) bytes of D) on
// the device.  For k_lz2 it is a copy of W whose end is congruent to the member's first chunk address modulo 16, so
// that W's tail and the chunk share 16-byte granules (stage_dict_chunk); null when the launch stages no history.
// win_len 0: the member has no dictionary.  dict_id: the Adler-32 of all of D (zlib's DICTID).
struct ZbMemberDict {
  const uint8_t *wend;
  uint32_t win_len, dict_id;
};
#define ZB_WIN_SLACK 16u   // bytes in front of each aligned copy of W (the bulk copies read whole 16-byte granules)
static inline uint32_t zb_win_stride(uint32_t win_len) { return ((win_len + 15u) & ~15u) + 3u * ZB_WIN_SLACK; }

// All device scratch for one compress batch (arrays sized by n_chunks / n_members).
struct ZbCompressWork {
  const uint8_t *src;          // device
  uint8_t *dst;                // device, 4-byte aligned; every byte of the output is written explicitly by k_pack
  uint64_t dst_cap;            // bytes (multiple of 4): a group that would end beyond this is not written at all
  const ZbChunkDesc *desc;     // [n_chunks]
  const uint32_t *member_first;// [n_members + 1] first chunk index of each member
  const uint8_t *fname_len;    // [n_members] gzip FNAME letters (0..25) or nullptr
  uint2 *masks;                // [n_chunks][2048] (token-start mask, is-match mask) per 32-byte window
  uint32_t *recs;              // [n_chunks][8 sub-chunks][2048] match records, one dense stream per sub-chunk
  uint16_t *hist;              // [n_chunks][8][316]
  ZbChunkCheck *chk;           // [n_chunks]
  ZbCodebook *cb;              // [n_chunks]
  uint64_t *chunk_off;         // [n_chunks] byte offset of each chunk's deflate bytes in dst
  uint64_t *member_off;        // [n_members + 1] output offsets (member_off[n] = total)
  uint32_t *member_check;      // [n_members] crc32 (gzip) or adler32 (zlib) of the whole member
  uint32_t *member_isize;      // [n_members] input size mod 2^32 (gzip ISIZE)
  const ZbMemberCarry *carry_in;  // [n_members] or null (= the empty prefix): folded in front of each member's chunks
  ZbMemberCarry *carry_out;       // [n_members] or null: carry_in followed by this launch's chunks
  uint64_t out_base;           // byte offset in dst where this group's first member starts ...
  const uint64_t *out_base_ptr;// ... or, when non-null, a device word holding it (the previous group's end),
                               // so consecutive groups can be enqueued without a host round trip
  const ZbCrcTables *tabs;     // device
  uint2 *lz2_tables;           // k_lz2 dictionaries: [grid][8 own tables of 2048 x 4 ways + 12 segment tables of 8192 entries], u16 positions (LZ levels only)
  uint32_t n_chunks, n_members;
  int level, data_format;
  // ZB_STRATEGY_*, after zb_strategy_level: RLE only at level 1 (k_lz<2>), FILTERED only at the LZ levels (k_lz2<false, 6>),
  // FIXED at any level but 0 (k_huff: stored or fixed blocks); HUFFMAN_ONLY never (it is level -2); OPTIMAL with
  // level 9 (k_opt instead of k_lz2)
  int strategy;
  // 2^window_bits (512..32768): no match reaches further back (k_lz<1>, k_lz2), and a zlib header's CINFO states it
  uint32_t max_dist;
  // Preset dictionaries (zb200_compress_batch_dicts and its k = 1 case, zb200_compress_batch_dict; a compress
  // stream's FDICT header): null, or [n_members] (group-relative, like desc[].member).  A member whose win_len is not
  // 0 gets FDICT and its dict_id in a zlib header; its first chunk, flagged ZB_CHUNK_DICT, stages its `pad` bytes of
  // history from wend (k_lz2).
  const ZbMemberDict *mdict;
  int dict_hist;               // some chunk is flagged ZB_CHUNK_DICT: the LZ levels run k_lz2<true>
  uint8_t *opt_scratch;        // strategy ZB_STRATEGY_OPTIMAL: k_opt's per-CTA chain links and path choices (zb_opt_scratch_bytes)
};

// per-device kernel attributes (dynamic shared memory limits); call with the device current
cudaError_t zb_setup_deflate_attrs();
cudaError_t zb_setup_inflate_attrs();
struct ZbLz2Params {
  uint32_t own_ways;   // ways of the own bucket looked at (1..4), after the closest same-hash position of the window
  uint32_t hist_segs;  // preceding segments whose entry is looked at (0..4), nearest first
  uint32_t maxcand;    // candidates per position that may pass the 4-byte check and be extended
  uint32_t good;       // a match this long leaves room for one more candidate only
  uint32_t lazy;       // matches shorter than this yield to a longer match at the next position (0: greedy)
  uint32_t max_dist;   // candidates at distance 1..max_dist are in the window (ZbCompressWork::max_dist)
};
// The level's effort under a window of max_dist bytes: a preceding segment j (0 = nearest) is looked at only when
// some of it can lie within max_dist, i.e. 8192 j < max_dist, so hist_segs is at most ceil(max_dist / 8192).
ZbLz2Params zb_lz2_params(int level, uint32_t max_dist);
size_t zb_lz2_table_bytes(int *grid_out);
// index_crc: the chunk checksums also hold the raw CRC-32 whatever the format (a compress-time index needs it)
cudaError_t zb_launch_lz(const ZbCompressWork &w, cudaStream_t s, bool index_crc = false);
cudaError_t zb_launch_huff(const ZbCompressWork &w, cudaStream_t s);
// the optimal parse (zb_optimal.cu): k_opt writes what k_lz2 writes; its scratch is opt_scratch, grid x (96 KiB of u16
// links + 64 KiB of u32 choices)
size_t zb_opt_scratch_bytes(int *grid_out);
cudaError_t zb_setup_opt_attrs();
cudaError_t zb_launch_opt(const ZbCompressWork &w, cudaStream_t s);
// rsyncable chunk map (zb_rsync.cu): member i is src[src_off[i], src_off[i + 1]); it is cut into tiles of
// ZB_RSYNC_MIN bytes, tiles tile_off[i] .. tile_off[i + 1] - 1 of the batch.  k_rsync_cand writes each tile's first
// and last gear-hash candidate into tile_cand; k_rsync_starts turns them into the member's chunk starts (member
// positions, ascending, the first 0) at starts + start_off[i] (start_off: prefix sums of zb_rsync_cap) and their
// number at counts[i].  Every array is device memory.
struct ZbRsyncWork {
  const uint8_t *src;
  const uint64_t *src_off, *tile_off, *start_off;   // [n + 1]
  uint32_t *tile_cand;                              // [n_tiles]
  uint64_t *counts;                                 // [n]
  uint64_t *starts;                                 // [start_off[n]]
  uint32_t n;
  uint64_t n_tiles;
};
cudaError_t zb_launch_rsync(const ZbRsyncWork &w, cudaStream_t s);
cudaError_t zb_launch_scan(const ZbCompressWork &w, cudaStream_t s);
cudaError_t zb_launch_pack(const ZbCompressWork &w, cudaStream_t s);
// A compress-time index (k_index_rec, after k_scan): the access-point records of zb200_index_build's recorder
// (ZbInflateWork::rec), taken from the block layout the compressor wrote instead of a decode.  A block start
// owns the multiples k * 32768 in (the previous block start's output offset, its own]; a member's first block owns
// k = 0.  For each owned k, record r = rec_first[member] + k - k0 receives rec[2r] = the bit position in the member,
// rec[2r + 1] = the member output offset; a block start that owns a multiple is a point, and crc[r] of its first
// one receives the CRC-32 of its interval (up to the next point or the member end) -- the raw (init 0) CRC
// instead when the interval runs past the end of a stream launch.  Records nobody owns stay as they were.
struct ZbIndexWork {
  uint64_t *rec;
  uint32_t *crc;
  const uint64_t *rec_first;   // [n_members] of the launch group
  uint64_t k0;                 // 0; a stream launch: the first multiple it can own
  uint64_t lo0;                // a stream launch that continues a member: the previous block start's output offset + 1
  uint64_t byte_base;          // a stream launch: the member bytes earlier launches wrote
  // [0]: the output offset of the launch's last block start; [1]: the raw CRC-32 of the output from the start of
  // a launch that continues a member up to its first point (or its end), 0 when that is empty (zeroed by the host)
  uint64_t *launch_out;
};
cudaError_t zb_launch_index_rec(const ZbCompressWork &w, const ZbIndexWork &x, cudaStream_t s);
// ---- inflate ----
struct ZbInflateWork {
  const uint8_t *src;          // device
  const uint64_t *src_off;     // device [n+1]
  uint8_t *dst;                // device (unused when count_only)
  const uint64_t *dst_off;     // device [n+1]; capacity of member i = dst_off[i+1]-dst_off[i]
  uint64_t *out_len;           // device [n]
  int *status;                 // device [n]
  uint32_t *expect;            // device [n] trailer checksum
  uint32_t *kind;              // device [n] resolved format (ZB_DF_*) per member
  uint32_t *counter;           // device work-queue counter (zeroed before launch)
  const ZbCrcTables *tabs;
  uint32_t n;
  int data_format;             // requested (may be ZB_DF_DETECT)
  uint64_t pos;                // payload start for raw ZB_DF_DEFLATE members (zb200_inflate's `pos`)
  int count_only;
  const uint32_t *order;       // device [n] or null: the work queue hands out members in this order (longest first)
  const uint8_t *skip;         // device [n] or null: members with skip[i] != 0 are left alone
  const uint64_t *seg_bits;    // device [2n] or null (seg_mode only): bit-exact (start, end) of segment i inside src --
                               //   speculative segments found by zb_launch_find_blocks; segment i > 0 may reference
                               //   32768 bytes before its own start (its unknown window)
  uint64_t seg_limit;          // with seg_bits: byte offset in src where the stream's payload ends
  int seg_win0;                // with seg_bits: segment 0 does not start the stream (a later window of a member):
                               //   it may reference 32768 bytes before its start too
  int mark;                    // with seg_bits: dst holds uint16 elements (dst_off in elements), 32768 marker
                               //   symbols sit in front of every segment's output
  int seg_mode;                // members are independently decodable SEGMENTS of one raw deflate stream:
                               // a segment also ends, successfully, when its input is used up at a block
                               // boundary; kind[i] reports whether a final block was seen
  // Gated queue (the host pipeline: ONE launch for a whole batch whose input is still arriving).  Queue
  // positions [gate_first[g], gate_first[g + 1]) belong to copy-in group g and are not started before
  // *gate_ready > g (written in stream order behind the group's copy); gate_done[g] counts the group's
  // finished members (a stream wait on it releases the group's copy-out).  Null: no gates.
  const uint32_t *gate_first;  // device [n_gates + 1]
  const uint32_t *gate_ready;  // device word
  uint32_t *gate_done;         // device [n_gates], zeroed before the launch
  uint32_t n_gates;
  // With seg_bits and count_only: null, or device [2] -- the last segment (n - 1) is then OPEN, the input a
  // decompress stream has received so far.  At every block start of that segment its lane 0 stores the block's
  // absolute bit position in src ([0]) and the segment's output count there ([1]).  When the segment stops with
  // ZB_ERR_END_OF_BUFFER (the input ran out) or ZB_ERR_DST_TOO_SMALL (the count ran out), its output up to [1] is
  // complete and the stream resumes decoding at bit [0].
  uint64_t *resume;
  // With seg_bits and count_only: null, or the access-point recorder of zb200_index_build.  rec_base [n + 1] (device)
  // holds every segment's output offset in the member.  Segment 0 owns the multiples k * 32768 in [0, rec_base[1]],
  // segment i > 0 those in (rec_base[i], rec_base[i + 1]]; for each owned k < nrec, rec[2k] / rec[2k + 1] receive the
  // bit position in src and the member output offset of the segment's first block start at or past the multiple.
  // A multiple that no block start of its segment reaches is left as it was (it belongs to the next segment's start).
  uint64_t *rec;
  const uint64_t *rec_base;
  uint32_t nrec;
  // Preset dictionaries (whole members only, not seg_bits): null, or [n] (indexed like src_off).  A raw member, or a
  // zlib member whose FDICT carries its dict_id, decodes as if its W were output in front of its first byte; gzip
  // members and zlib members without FDICT ignore it.  A member with win_len 0 decodes as without a dictionary.
  const ZbMemberDict *mdict;
};
cudaError_t zb_launch_inflate(const ZbInflateWork &w, cudaStream_t s);
// positions just past every byte sequence 00 00 ff ff (the empty stored block that byte-aligns a
// stream: zlib's sync / full flush, and the joint between this library's 64 KiB chunks) inside
// src[lo, hi): unordered, *count may exceed cap (then the list is incomplete)
cudaError_t zb_launch_find_sync(const uint8_t *src, uint64_t lo, uint64_t hi, uint64_t *out, uint32_t cap,
                                uint32_t *count, cudaStream_t s);

// candidate starts (bit positions) of dynamic deflate blocks inside src bits [lo_bit, hi_bit): unordered,
// *count may exceed cap; bytes at and beyond limit_byte read as zero
cudaError_t zb_launch_find_blocks(const uint8_t *src, uint64_t lo_bit, uint64_t hi_bit, uint64_t limit_byte, uint64_t *out,
                                  uint32_t cap, uint32_t *count, cudaStream_t s);
// speculative segments decoded as uint16 symbols (ZbInflateWork::mark): marker prefill and resolution
struct ZbMarkSegHost {
  uint64_t scr;   // element offset of the segment's first output symbol in the scratch
  uint64_t dst;   // byte offset of the segment's first output byte in dst
  uint32_t n;     // output bytes
  uint32_t pad;
};
cudaError_t zb_launch_mark_prefill(uint16_t *scr, const void *segs, uint32_t nseg, cudaStream_t s);
// base: dst offset of the member's first output byte
cudaError_t zb_launch_resolve(const uint16_t *scr, const void *segs, uint32_t nseg, uint32_t max_n, uint64_t base, uint8_t *dst,
                              int *bad, cudaStream_t s);
// The parallel window resolve (zb_resolve.h): the segments are one window of a member, in groups of gsz; w0 is the
// member position of the window's first byte (the resolved output in front of it is in dst already).  Scratch:
// gmap [ceil(nseg / gsz) x 32768] uint16, gin the same count of bytes.  Rewrites the tails in scr.
cudaError_t zb_launch_resolve_groups(uint16_t *scr, const void *segs, uint32_t nseg, uint32_t max_n, uint32_t gsz, uint64_t base,
                                     uint64_t w0, uint16_t *gmap, uint8_t *gin, uint8_t *dst, int *bad, cudaStream_t s);

// byte ranges copied from src to dst, at most ZB_GATHER_BYTES each; wide: dst is uint16 symbols (a window placed
// in the marker scratch, each byte its own literal symbol) and dst counts elements
#define ZB_GATHER_BYTES 65536u
struct ZbGather {
  uint64_t src;
  uint64_t dst;
  uint32_t n;
  uint32_t wide;
};
cudaError_t zb_launch_gather(const uint8_t *src, const ZbGather *g, uint32_t n, void *dst, cudaStream_t s);

// ---- checksums over a batch of buffers (standalone crc32/adler32, and the trailer
// verification after inflate) ----
#define ZB_CK_PIECE_BYTES 32768   // the checksum kernels cut every buffer into pieces of this size
struct ZbPiece {
  uint64_t rel;   // start of the piece relative to its buffer
  uint32_t buf;   // buffer index
  uint32_t pad;
};
struct ZbChecksumWork {
  const uint8_t *src;          // device: base of the buffers
  const uint64_t *off;         // device [n+1]: buffer i starts at src + off[i]
  const uint64_t *lens;        // device [n] actual lengths, or null (= off[i+1]-off[i])
  const ZbPiece *pieces;       // device [n_pieces]: ZB_CK_PIECE_BYTES pieces covering every buffer's capacity
  const uint32_t *first;       // device [n+1]: first piece of each buffer
  ZbChunkCheck *piece_out;     // device [n_pieces] scratch
  uint32_t *partials;          // device [n_pieces * 512] scratch: the CRC path's per-warp, per-lane words of full pieces
  uint32_t *out;               // device [n] checksums, or null
  int *status;                 // device [n] or null: buffers with a non-zero status are skipped;
                               //   verify mode writes ZB_ERR_CHECKSUM / ZB_ERR_SIZE here
  const uint32_t *expect;      // device [n] expected value (verify mode) or null
  const uint32_t *kinds;       // device [n] resolved ZB_DF_* per buffer (gzip -> crc32, zlib -> adler32) or null
  const uint8_t *isize_src;    // verify mode: compressed buffers (gzip ISIZE lives in their last 4 bytes)
  const uint64_t *isize_off;   //   and their offsets [n+1]
  const ZbCrcTables *tabs;
  uint32_t n, n_pieces;
  int kind;                    // 0 crc32, 1 adler32 when kinds == null
  uint32_t big_pieces;         // 0, or: buffers of more pieces than this are folded by a whole CTA (k_buffer_combine_big)
                               //   instead of one warp (the host sets it when some buffer's capacity is that large)
};
#define ZB_CK_BIG_PIECES 2048u  // 64 MiB
#define ZB_CK_PARTIAL_BYTES 2048  // per piece in ZbChecksumWork::partials
cudaError_t zb_launch_checksum(const ZbChecksumWork &w, cudaStream_t s);
