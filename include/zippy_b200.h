/*
 * zippy_b200.h -- C ABI of libzippy_b200.so, the H100 (sm_90a) replacement for the codec
 * core of guzba/zippy.  Plain pointers and sizes only; no CUDA or torch types.
 *
 * The four single-input entry points are exactly the seam the reference's framing layer
 * calls (SURVEY.md section 8b):
 *     zb200_deflate  <->  proc deflate*(dst: var string, src, len, level)   src/zippy/deflate.nim:207
 *     zb200_inflate  <->  proc inflate*(dst: var string, src, len, pos)     src/zippy/inflate.nim:268
 *     zb200_crc32    <->  proc crc32*(src: pointer, len: int): uint32       src/zippy/crc.nim:53
 *     zb200_adler32  <->  proc adler32*(src: pointer, len: int): uint32     src/zippy/adler32.nim:6
 * The batch entry points have no reference counterpart (the reference is one input per
 * call); they are what makes a GPU worthwhile and what zippy.compress/uncompress map onto
 * when a caller has many inputs (e.g. ziparchives.nim:505-540 createZipArchive's loop).
 *
 * Conventions
 *  - every function returns a ZB200_* status (0 = ok) unless documented otherwise;
 *    statuses mirror the reference's ZippyError messages one to one (zb200_strerror).
 *  - the library never keeps or frees caller memory; `dst` buffers are caller-allocated
 *    (zb200_*_bound gives a sufficient size).
 *  - a zb200_ctx is bound to one CUDA device and one stream; calls on the same ctx
 *    serialise, different ctxs may be used from different host threads.
 *  - there is no CPU fallback: without a CUDA device zb200_init fails with ZB200_ERR_CUDA.
 */
#ifndef ZIPPY_B200_H
#define ZIPPY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* status codes; 1..18 are the reference's ZippyError messages (SURVEY.md 8b "Error convention") */
enum {
  ZB200_OK = 0,
  ZB200_ERR_INVALID_LEVEL = 1,   /* "Invalid compression level"             deflate.nim:209 */
  ZB200_ERR_INVALID_FORMAT = 2,  /* "Invalid data format"                   zippy.nim:84 */
  ZB200_ERR_UNCOMPRESS = 3,      /* "Invalid buffer, unable to uncompress"  internal.nim:191 */
  ZB200_ERR_COMPRESS = 4,        /* "Unexpected error while compressing"    internal.nim:194 */
  ZB200_ERR_END_OF_BUFFER = 5,   /* "Cannot read further, at end of buffer" bitstreams.nim:16 */
  ZB200_ERR_BYTE_BOUNDARY = 6,   /* "Must be at a byte boundary"            bitstreams.nim:66 */
  ZB200_ERR_BLOCK_HEADER = 7,    /* "Invalid block header"                  inflate.nim:289 */
  ZB200_ERR_INVALID_SYMBOL = 8,  /* "Invalid symbol"                        inflate.nim:165 */
  ZB200_ERR_DETECT = 9,          /* "Unable to detect compressed data format" zippy.nim:125 */
  ZB200_ERR_METHOD = 10,         /* "Unsupported compression method"        zippy.nim:141 */
  ZB200_ERR_CINFO = 11,          /* "Invalid compression info"              zippy.nim:144 */
  ZB200_ERR_HEADER = 12,         /* "Invalid header"                        zippy.nim:147 */
  ZB200_ERR_FDICT = 13,          /* "Preset dictionary is not yet supported" zippy.nim:150 */
  ZB200_ERR_CHECKSUM = 14,       /* "Checksum verification failed"          zippy.nim:162, gzip.nim:81 */
  ZB200_ERR_GZIP_ID = 15,        /* "Failed gzip identification values check" gzip.nim:23 */
  ZB200_ERR_GZIP_RESERVED = 16,  /* "Reserved flag bits set"                gzip.nim:29 */
  ZB200_ERR_GZIP_FLAGS = 17,     /* "Currently unsupported flags are set"   gzip.nim:41 */
  ZB200_ERR_SIZE = 18,           /* "Size verification failed"              gzip.nim:85 */
  /* new classes with no reference counterpart */
  ZB200_ERR_DST_TOO_SMALL = 19,
  ZB200_ERR_CUDA = 20,
  ZB200_ERR_NOMEM = 21,
  ZB200_ERR_ARG = 22,
  ZB200_ERR_DICTIONARY = 23      /* a zlib member's DICTID is not the Adler-32 of the dictionary given */
};

/* CompressedDataFormat (src/zippy/common.nim:4-5), same ordinals */
enum { ZB200_DF_DETECT = 0, ZB200_DF_ZLIB = 1, ZB200_DF_GZIP = 2, ZB200_DF_DEFLATE = 3 };
/* levels (src/zippy/common.nim:7-12) */
enum { ZB200_NO_COMPRESSION = 0, ZB200_BEST_SPEED = 1, ZB200_BEST_COMPRESSION = 9,
       ZB200_DEFAULT_COMPRESSION = -1, ZB200_HUFFMAN_ONLY = -2 };

typedef struct zb200_ctx zb200_ctx;

/* ---- lifecycle ---- */
int zb200_init(int device, zb200_ctx **out);  /* device < 0: current device */
void zb200_shutdown(zb200_ctx *ctx);
const char *zb200_strerror(int status);       /* the reference's message for 1..18 */
const char *zb200_last_cuda_error(zb200_ctx *ctx);
/* run this ctx's work on a caller-owned CUDA stream (a cudaStream_t passed as void*;
 * NULL restores the ctx's own stream) so callers can order and time it with their events */
int zb200_set_stream(zb200_ctx *ctx, void *cuda_stream);
int zb200_device_count(void);

/* ---- sizing ---- */
/* bound on raw-deflate bytes for `len` input bytes (stored path + per-block overhead;
 * the reference itself grows its output, bitstreams.nim:96-98) */
size_t zb200_deflate_bound(size_t len);
/* bound including the gzip (<= 36 + 8 bytes) / zlib (2 + 4) framing of zippy.nim:21-78 */
size_t zb200_compress_bound(size_t len, int data_format);

/* ---- single input, host buffers (the reference seam) ---- */
/* deflate.nim:207: raw RFC1951 stream, BFINAL on the last block, byte aligned at the end */
int zb200_deflate(zb200_ctx *ctx, const uint8_t *src, size_t len, int level,
                  uint8_t *dst, size_t dst_cap, size_t *dst_len);
/* inflate.nim:268: decode the raw stream that starts at byte `pos` of src[0..len) */
int zb200_inflate(zb200_ctx *ctx, const uint8_t *src, size_t len, size_t pos,
                  uint8_t *dst, size_t dst_cap, size_t *dst_len);
/* size the output of zb200_inflate without producing it */
int zb200_inflate_size(zb200_ctx *ctx, const uint8_t *src, size_t len, size_t pos, size_t *out_len);
/* One input whose output size is unknown, decoded ONCE: begin inflates (and verifies the trailer) into
 * library-owned device memory and reports the size, finish copies the bytes out.  This is what a caller
 * with a growing destination (the reference's `dst: var string`, inflate.nim:268-291, gzip.nim:3-88) binds
 * instead of inflate_size + inflate (two decodes).  data_format as for uncompress; `pos` as for inflate
 * (raw streams only).  A gzip member whose ISIZE understates its content gets the reference's verdict
 * (data, CRC check, then "Size verification failed"), not "destination too small". */
int zb200_decode_begin(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, size_t pos, size_t *out_len);
int zb200_decode_finish(zb200_ctx *ctx, uint8_t *dst, size_t dst_cap, size_t *dst_len);
/* crc.nim:53 / adler32.nim:6 */
int zb200_crc32(zb200_ctx *ctx, const void *src, size_t len, uint32_t *out);
int zb200_adler32(zb200_ctx *ctx, const void *src, size_t len, uint32_t *out);

/* ---- batches of independent inputs, host buffers ----
 * input i is src_base[src_offsets[i] .. src_offsets[i+1]); offsets arrays have n+1 entries.
 * compress: zippy.compress(src, level, dataFormat) per input (zippy.nim:11-84); output i is
 * written at dst_base[dst_offsets[i] .. dst_offsets[i+1]) with dst_offsets filled in.
 * fname_lens (gzip only, may be NULL = all 0): number of 'a'.. letters the reference draws
 * at random for the FNAME field (zippy.nim:28-42); each in 0..25. */
int zb200_compress_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                         int level, int data_format, const uint8_t *fname_lens,
                         uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
/* uncompressed size of every input (gzip: ISIZE trailer, gzip.nim:66; zlib/raw: a counting
 * pass over the stream).  sizes[i] is only meaningful where statuses[i] == 0. */
int zb200_uncompress_sizes(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           int data_format, uint64_t *sizes, int *statuses);
/* zippy.uncompress(src, dataFormat) per input (zippy.nim:100-165).  dst_offsets (n+1, in)
 * gives each output's slot; slot capacity is dst_offsets[i+1]-dst_offsets[i]; dst_lens[i]
 * receives the produced size.  A failing input sets statuses[i] and produces no output.
 * Members are independent and decoded in parallel; ONE member is a serial stream (one 8-lane group, ~10 MB/s),
 * so members of 512 KiB or more are first cut into parallel segments: at every byte-aligning empty stored
 * block 00 00 ff ff when the stream has them (this library's own multi-chunk output, zlib full-flush streams),
 * otherwise at dynamic-block starts found by testing every bit offset, each segment decoded with marker symbols
 * for its unknown 32 KiB window and resolved afterwards (any gzip / zlib output).  The serial decode is the
 * fallback for anything irregular -- results, including the error reported, are identical either way.
 * Limits: on the serial path one member's output is at most 4 GiB - 33 KiB (32-bit positions inside a member);
 * members decoded as segments have no such limit.
 * With page-locked host buffers the copies in and out overlap the kernels (member groups); pageable buffers
 * are staged through an internal pinned ring. */
int zb200_uncompress_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           int data_format, uint8_t *dst_base, const uint64_t *dst_offsets,
                           uint64_t *dst_lens, int *statuses);
/* zb200_uncompress_batch(..., ZB200_DF_DEFLATE, ...) -- the same slots, statuses and outputs -- that also
 * returns crcs[i], the CRC-32 of output i, wherever statuses[i] == 0 (0 elsewhere).  The CRC is computed on the
 * device from the decoded bytes, in the pass that verifies gzip / zlib trailers; raw deflate has no trailer, so
 * nothing is compared.  For containers that keep each entry's CRC-32 in their headers (ZIP). */
int zb200_inflate_batch_crc32(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                              uint8_t *dst_base, const uint64_t *dst_offsets, uint64_t *dst_lens, uint32_t *crcs,
                              int *statuses);
/* ---- preset dictionaries (zlib's deflateSetDictionary / inflateSetDictionary, Python zlib's zdict) ----
 * D = dict[0 .. dict_len), any length; the window W is its last min(32768, dict_len) bytes and DICTID is the
 * Adler-32 of all of D.  dict_len == 0 is exactly the call without a dictionary (outputs and statuses).
 * Dictionaries apply to zlib and raw DEFLATE; D is uploaded once per call and shared by every member.
 *  - compress: a zlib member starts 78 20 DICTID (big-endian), so it is 4 bytes longer than without a dictionary
 *    (bound: zb200_compress_bound(len, fmt) + 4); its trailer is the Adler-32 of the input alone.  At levels -1 and
 *    2..9 the member's first chunk sees W as its history: the blocks are byte for byte what a compress stream of the
 *    same level emits for the input after W was written and sync-flushed.  Levels 0, 1 and -2 keep no history:
 *    their blocks are those without a dictionary.  gzip with a non-empty dictionary: ZB200_ERR_INVALID_FORMAT.
 *  - decode: a raw stream S decodes (output and status) as uncompress(stored(W) || S, DEFLATE) without its first
 *    |W| output bytes, stored(W) being the one non-final stored block 00 LEN ~LEN W: a distance may reach |W| bytes
 *    in front of the output.  A zlib member with FDICT: ZB200_ERR_FDICT without a dictionary (dict_len 0, or the
 *    calls without _dict), ZB200_ERR_UNCOMPRESS below 10 bytes, ZB200_ERR_DICTIONARY if its DICTID is not D's,
 *    else its payload from byte 6 decodes as a raw stream above and the trailer is checked against the Adler-32 of
 *    the output.  gzip members and zlib members without FDICT ignore the dictionary; DETECT works as without one.
 *  - uncompress_batch_dict decodes every member whole, one 8-lane group per member (~10 MB/s each): members of
 *    512 KiB and more are not cut into parallel segments.  decode_begin_dict (finished by zb200_decode_finish; raw
 *    members start at byte 0) decodes stored(W) || payload through zb200_decode_begin's paths, so large members
 *    decode in parallel wherever they do without a dictionary.
 *  - compress_stream_begin_dict: a compress stream (below) whose history starts as W (LZ levels) and whose zlib
 *    header carries DICTID; a full flush drops W with the rest of the history.  No FNAME: gzip is refused. */
int zb200_compress_batch_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                              int level, int data_format, const uint8_t *dict, size_t dict_len,
                              uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_uncompress_sizes_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int data_format, const uint8_t *dict, size_t dict_len, uint64_t *sizes, int *statuses);
int zb200_uncompress_batch_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int data_format, const uint8_t *dict, size_t dict_len, uint8_t *dst_base,
                                const uint64_t *dst_offsets, uint64_t *dst_lens, int *statuses);
int zb200_decode_begin_dict(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, const uint8_t *dict,
                            size_t dict_len, size_t *out_len);
/* ---- per-member preset dictionaries: a table of k dictionaries, one entry (or none) per member ----
 * Entry j is dict_base[dict_offsets[j] .. dict_offsets[j + 1]) (dict_offsets has k + 1 entries); member i uses
 * entry dict_of[i], -1 for none.  Let D be member i's entry (W, DICTID as above) and M its input.  Members may
 * share an entry: its DICTID is computed and its bytes uploaded once per call.  The *_dict calls are the k = 1
 * case with every dict_of[i] = 0, and write and decode exactly what these calls do for that table.
 *  - compress, window_bits 15: a member with a non-empty D is byte for byte zb200_compress_batch_dict(M alone, D);
 *    one with dict_of[i] == -1 or an empty D is byte for byte zb200_compress_batch(M alone).  A member's bytes do
 *    not depend on the other members, its position in the batch or how the table is shared.
 *  - compress, window_bits n in 9..15 (validated as in zb200_compress_batch_window: 8 means 9 for zlib): a member
 *    without a dictionary is zb200_compress_batch_window(M alone) at n.  A member with D: its blocks are byte for
 *    byte what a raw compress stream of the same level and window_bits n writes for M after D was written to it and
 *    sync-flushed; no match reaches more than 2^n bytes back, into M or into W (W stays the last
 *    min(32768, |D|) bytes of D); a zlib header is CMF (n - 8) << 4 | 8, FLG with FDICT, FLEVEL 0 and FCHECK, then
 *    the DICTID.  Levels 0, 1 and -2 keep no history: only their header carries D.
 *  - bound: zb200_compress_bound(len, fmt) + 4 for every zlib member with a non-empty D.
 *  - decode: a member decodes (output, size, status) exactly as zb200_uncompress_batch_dict / _sizes_dict do with
 *    its D alone; a member with -1 as zb200_uncompress_batch / _sizes (FDICT: ZB200_ERR_FDICT).  A DICTID that is
 *    not D's: ZB200_ERR_DICTIONARY.  gzip members and zlib members without FDICT ignore the entry they name;
 *    DETECT works as with _dict.  A batch in which some member names a non-empty D decodes every member whole, as
 *    uncompress_batch_dict does.
 *  - whole-call errors, statuses left alone: ZB200_ERR_ARG for a dict_of outside -1 .. k - 1, dict_offsets that
 *    decrease, or a null dict_of with n > 0; ZB200_ERR_INVALID_FORMAT for a gzip compress in which a member names
 *    a non-empty D.
 *  - limits: windows go to the device with their launch group and their memory is bounded by the groups in flight,
 *    not by the batch: a group holds one copy of W (|W| rounded up to 16, plus 48 bytes) per (entry, member address
 *    modulo 16) its members use (decode: per entry), three groups' worth at a time (a decode keeps every group's
 *    windows, in one launch, only while they fit that much); a decode group holds at most 256 MiB of windows.  The
 *    DICTIDs of named entries above 256 KiB in all are computed on the device, from uploads of at most 256 MiB of
 *    consecutive named entries at a time (an entry larger than that alone).  Plus 16 bytes per member. */
int zb200_compress_batch_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                               int level, int data_format, int window_bits,
                               const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k, const int32_t *dict_of,
                               uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_uncompress_sizes_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                                 const int32_t *dict_of, uint64_t *sizes, int *statuses);
int zb200_uncompress_batch_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                                 const int32_t *dict_of, uint8_t *dst_base, const uint64_t *dst_offsets,
                                 uint64_t *dst_lens, int *statuses);

/* crc32 (kind 0) or adler32 (kind 1) of every input */
int zb200_checksum_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                         int kind, uint32_t *out);

/* ---- streaming compression: one gzip / zlib / raw member from input that arrives piece by piece ----
 * What a stream emits, concatenated, is byte for byte what zb200_compress_batch writes for the whole input as
 * one member (same level, format and fname_len), whatever the sizes of the writes.
 *  - begin: level -2..9, data_format GZIP / ZLIB / DEFLATE, fname_len 0..25 (gzip FNAME letters, as
 *    fname_lens in compress_batch; ignored for the other formats).  An invalid level or format fails with
 *    ZB200_ERR_INVALID_LEVEL / ZB200_ERR_INVALID_FORMAT, an invalid fname_len with ZB200_ERR_ARG.
 *  - The stream's state lives on the host inside the stream object: the pending input, the last 32 KiB of
 *    input already compressed (the LZ levels' history), the running CRC-32 / Adler-32 and 64-bit byte count,
 *    whether the header went out.  There is no device memory per stream; the kernels use the ctx's scratch.
 *    Several streams may be open on one ctx, interleaved with each other and with any other call on it; calls
 *    on one ctx serialise as always.  Free every stream of a ctx before zb200_shutdown.
 *  - Chunking is the one-shot call's: 64 KiB chunks from the start of the member.  A chunk is compressed only
 *    once it is known not to be the last, so a stream always holds back 1..65536 bytes (none only when nothing
 *    was written); finish compresses what is held back as the last chunk, then writes the trailer.  A stream
 *    with no input finishes as the empty member.  The header goes out with the first emitted bytes.
 *  - write launches kernels only once a batch of input is pending (64 MiB, tools/bench_compress_stream.py);
 *    smaller writes are only buffered and emit nothing.  *dst_len receives what was emitted.
 *  - bound(st, len): the most bytes the next write of `len` bytes (or finish: len = 0) can emit.
 *  - A write or finish after finish: ZB200_ERR_ARG.  ZB200_ERR_DST_TOO_SMALL consumes nothing and leaves the
 *    stream as it was: retry with bound() bytes.  After a CUDA failure every later call reports it.
 *  - Members of 4 GiB and more work: the byte count is 64-bit, gzip ISIZE is the total mod 2^32.
 *  - flush(st, mode): emit everything written so far (the header too if it has not gone out), so that every byte
 *    written can be decoded from what has been emitted.  mode is ZB200_SYNC_FLUSH or ZB200_FULL_FLUSH (zlib's
 *    Z_SYNC_FLUSH / Z_FULL_FLUSH); anything else, or a flush after finish: ZB200_ERR_ARG.  The flush offsets cut
 *    the member into flush segments, each cut into 64 KiB chunks from its own start; a segment's last chunk may be
 *    short and ends, like every chunk but the member's last, in the byte-aligning empty stored block 00 00 ff ff.
 *    Levels -1 and 2..9 see min(32 KiB, bytes since the member start or the last FULL flush) of history: a sync
 *    flush keeps the history, a full flush drops it (no match reaches back across it, and a raw inflater started
 *    right after it decodes the rest).  Levels 0, 1 and -2 have no history, so both modes write the same bytes.
 *    The member's bytes depend only on the input, the flush offsets and modes, level, format and fname_len --
 *    never on the write sizes or the batching threshold.  Without a flush, or with sync flushes only at multiples
 *    of 64 KiB, they are compress_batch's bytes.  A flush with nothing written since the last flush (or begin)
 *    emits nothing and changes nothing; finish right after a flush writes the empty final block (03 00, at
 *    level 0 the empty stored block) and the trailer.  bound(st, 0) also bounds what a flush emits;
 *    ZB200_ERR_DST_TOO_SMALL and CUDA failures behave as for write.
 *  - free: at any time, finished or not. */
enum { ZB200_SYNC_FLUSH = 2, ZB200_FULL_FLUSH = 3 };
typedef struct zb200_compress_stream zb200_compress_stream;
int zb200_compress_stream_begin(zb200_ctx *ctx, int level, int data_format, int fname_len, zb200_compress_stream **out);
int zb200_compress_stream_begin_dict(zb200_ctx *ctx, int level, int data_format, const uint8_t *dict, size_t dict_len,
                                     zb200_compress_stream **out);
size_t zb200_compress_stream_bound(const zb200_compress_stream *st, size_t len);
int zb200_compress_stream_write(zb200_compress_stream *st, const uint8_t *src, size_t len,
                                uint8_t *dst, size_t dst_cap, size_t *dst_len);
int zb200_compress_stream_flush(zb200_compress_stream *st, int mode, uint8_t *dst, size_t dst_cap, size_t *dst_len);
int zb200_compress_stream_finish(zb200_compress_stream *st, uint8_t *dst, size_t dst_cap, size_t *dst_len);
void zb200_compress_stream_free(zb200_compress_stream *st);

/* ---- streaming decompression: one gzip / zlib / raw member from compressed input that arrives piece by piece ----
 * Whatever the sizes of the writes (empty ones included), everything read from a stream, concatenated, is
 * byte for byte what zippy.uncompress(whole input, data_format) returns, and the stream's final status is that
 * call's status.  One exception: a member whose output exceeds 4 GiB - 33 KiB and that uncompress can only decode
 * serially (no parallel segments) ends there with ZB200_ERR_DST_TOO_SMALL; a stream has no such limit and decodes it.
 *  - begin: data_format DETECT, GZIP, ZLIB or DEFLATE (anything else: ZB200_ERR_INVALID_FORMAT).  Raw streams
 *    start at byte 0 (there is no `pos`).
 *  - write consumes all of src; *avail (may be NULL) receives the decoded bytes now waiting to be read.  finish
 *    says the input has ended: it decodes what is held, then checks the trailer, checksum before size.
 *    read moves up to dst_cap waiting bytes into dst (*dst_len: how many); it works after finish too.
 *  - What depends on the input's length waits until the length is known: nothing about the header is decided
 *    before 19 bytes have arrived (or finish), and the last 8 (gzip) / 4 (zlib) bytes are always held back as the
 *    possible trailer.  As in uncompress, bytes between the final block and the trailer are ignored, and so is
 *    anything after a raw stream's final block.  A second gzip member is not decoded (the reference rejects it).
 *  - Errors: once a write or finish fails, every later call (read included) returns the same status.  Bytes read
 *    before that come only from blocks that decoded completely; for a truncated member they are a prefix of its
 *    output.  A write or finish after finish: ZB200_ERR_ARG.
 *  - The stream's state lives on the host inside the stream object: the compressed input not decoded yet (from a
 *    block boundary on), the last 32 KiB of output, the running CRC-32 / Adler-32 and 64-bit output count (ISIZE is
 *    compared mod 2^32), the wrapper, the decoded bytes not read yet.  There is no device memory per stream; the
 *    kernels use the ctx's scratch.  Several streams may be open on one ctx, interleaved with each other and with any
 *    other call on it; calls on one ctx serialise as always.  Free every stream of a ctx before zb200_shutdown.
 *  - write launches kernels only once a batch of compressed input is pending (64 MiB,
 *    tools/bench_decompress_stream.py); smaller writes are only buffered.  One launch reads at most twice that much
 *    input and produces at most about 1 GiB (more only when a single block is larger); a large write is decoded by
 *    as many launches as it needs before it returns.
 *  - drain decodes now, whatever the batching threshold, every block that is complete in the input received so
 *    far, and *avail (may be NULL) receives the bytes waiting to be read.  A block that ends inside the bytes held
 *    back as the possible trailer counts too, so after a sender's sync or full flush (this library's, zlib's) a
 *    drain yields everything written up to it.  If the input does end there, the member has no final block
 *    before its trailer and finish reports uncompress's error.  Before the header is decided (19 member bytes,
 *    and for gzip the whole header and 9 bytes more) drain decodes nothing.  As for write, an error in a block that starts
 *    less than 1 KiB before the end of the input so far is only believed at finish.  drain after finish:
 *    ZB200_ERR_ARG; a failure is the stream's error, as for write.
 *  - Decoded bytes stay in the stream until read: read after every write or drain.
 *  - free: at any time, finished or not. */
typedef struct zb200_decompress_stream zb200_decompress_stream;
int zb200_decompress_stream_begin(zb200_ctx *ctx, int data_format, zb200_decompress_stream **out);
/* a decompress stream against a preset dictionary (see "preset dictionaries" above): what it returns, and its status,
 * are zb200_decode_begin_dict's for the whole input.  A raw stream, or a zlib member whose FDICT carries D's DICTID,
 * holds stored(W) in front of its payload once the header is decided; the window's bytes are never returned or
 * checksummed.  gzip members and zlib members without FDICT ignore the dictionary. */
int zb200_decompress_stream_begin_dict(zb200_ctx *ctx, int data_format, const uint8_t *dict, size_t dict_len,
                                       zb200_decompress_stream **out);
int zb200_decompress_stream_write(zb200_decompress_stream *st, const uint8_t *src, size_t len, size_t *avail);
int zb200_decompress_stream_drain(zb200_decompress_stream *st, size_t *avail);
int zb200_decompress_stream_finish(zb200_decompress_stream *st, size_t *avail);
int zb200_decompress_stream_read(zb200_decompress_stream *st, uint8_t *dst, size_t dst_cap, size_t *dst_len);
void zb200_decompress_stream_free(zb200_decompress_stream *st);

/* ---- random access into one gzip / zlib / raw member (a seekable index, as zlib's zran.c builds on a CPU) ----
 * build decodes the member once, with uncompress's verdict (any failure is returned and no index is made), and
 * records access points.  Segment points: for k = 0, 1, ..., the first block start whose output offset is at least
 * k * 32768 (duplicates removed; point 0 is the first block, at offset 0).  Window points: for j = 0, 1, ..., the
 * first segment point at or past j * span; each keeps the 32 KiB of output in front of it.  Every segment point keeps
 * the CRC-32 of its interval (to the next point; the last one to the end of the member).  The points depend only on
 * the member.  Random access is only as fine as the member's blocks: this library's members have a point at every
 * 64 KiB chunk joint, zlib's at its block starts, and a member of one block has one point.
 *  - build: span a multiple of 32768 and >= 32768 (zran's usual span is 1 << 20), else ZB200_ERR_ARG; a bad
 *    data_format: ZB200_ERR_INVALID_FORMAT.  The index is host memory and belongs to no ctx: use it with any ctx,
 *    from any thread, and free it with zb200_index_free.
 *  - extract_batch reads the n ranges [offsets[i], offsets[i] + lens[i]) of the member's output into
 *    dst[dst_offsets[i] ..) (dst_offsets has n + 1 entries; slot i holds dst_offsets[i+1] - dst_offsets[i] bytes).
 *    ZB200_ERR_ARG, before any work: src's length or its first or last 32 bytes differ from the indexed member, a
 *    range ends past the output, or a slot is too small.  Ranges may be empty and may overlap.  Every range is cut
 *    at window points; each piece is decoded from its window point through the intervals it needs, and all of these
 *    chains run in parallel, in launch groups of about 1 GiB of output.  Only the compressed bytes the chains cover
 *    cross PCIe, with their windows.  statuses[i]: ZB200_OK with the exact bytes, ZB200_ERR_UNCOMPRESS if an
 *    interval it needs does not decode to its recorded size and end, ZB200_ERR_CHECKSUM if it decodes but its CRC-32
 *    differs (the gzip / zlib trailer is not read).
 *  - points copies min(cap, count) points out (any array may be NULL) and returns the count.
 *  - export writes the index as bytes (dst == NULL: only *len, the size); the same member and span give the same
 *    bytes on any run and any ctx.  import reads them back; anything malformed (wrong length, magic, version or
 *    CRC, counts that do not fit, points not strictly increasing in bit and output offset, a window flag that
 *    breaks the rule above, a window that does not decompress to exactly 32768 bytes) is ZB200_ERR_ARG, and
 *    nothing is read out of bounds.  Format, all integers little-endian:
 *      offset  size  field
 *           0     8  magic "ZB200IDX"
 *           8     4  version (1)
 *          12     4  data format (ZB200_DF_ZLIB / _GZIP / _DEFLATE, as resolved by the build)
 *          16     8  payload start P (byte offset of the raw DEFLATE stream in the member)
 *          24     8  member length in bytes
 *          32     8  output size
 *          40     8  span
 *          48     8  reserved (0)
 *          56    32  the member's first 32 bytes (zero-padded if shorter)
 *          88    32  the member's last 32 bytes (zero-padded if shorter)
 *         120     8  np: number of segment points (>= 1)
 *         128     8  nw: number of windows (window points with output offset > 0)
 *         136  24np  per point: bit position in the member (8), output offset (8), interval CRC-32 (4), window flag (4)
 *           .   8nw  per window: length of its compressed form
 *           .     .  the windows in point order, each the raw DEFLATE (level 1) of the 32768 bytes in front of its point
 *           .     4  CRC-32 of every byte before it */
typedef struct zb200_index zb200_index;
int zb200_index_build(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, uint64_t span, zb200_index **out);
int zb200_index_extract_batch(zb200_ctx *ctx, const zb200_index *idx, const uint8_t *src, size_t len,
                              const uint64_t *offsets, const uint64_t *lens, size_t n, uint8_t *dst,
                              const uint64_t *dst_offsets, int *statuses);
uint64_t zb200_index_size(const zb200_index *idx);   /* the member's output size */
size_t zb200_index_points(const zb200_index *idx, uint64_t *bits, uint64_t *outs, uint32_t *crcs, uint8_t *window,
                          size_t cap);
void zb200_index_free(zb200_index *idx);
int zb200_index_export(zb200_ctx *ctx, const zb200_index *idx, uint8_t *dst, size_t cap, size_t *len);
int zb200_index_import(zb200_ctx *ctx, const uint8_t *src, size_t len, zb200_index **out);

/* ---- an index written while compressing (no decode pass) ----
 * zb200_compress_batch_index / zb200_compress_batch_device_index take zb200_compress_batch's /
 * zb200_compress_batch_device's arguments plus span and indexes (n entries), and write the same members as those
 * calls.  indexes[i] receives a new index of member i (free it with zb200_index_free) that exports to exactly the
 * bytes zb200_index_build(member i, data_format, span) + zb200_index_export give, or NULL where statuses[i] != 0
 * (every entry is NULL when the call fails).  The points come from the block layout the compressor wrote, the
 * interval CRC-32s from the chunk checksums, the windows from the input.
 * zb200_compress_stream_begin_index begins a stream as zb200_compress_stream_begin does that also writes the index;
 * zb200_compress_stream_index, valid only after zb200_compress_stream_finish on such a stream (anything else is
 * ZB200_ERR_ARG), returns a new index of the whole member.  span: a multiple of 32768, at least 32768, else
 * ZB200_ERR_ARG before any work; an invalid level or format is reported as by the calls without an index. */
int zb200_compress_batch_index(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                               int data_format, const uint8_t *fname_lens, uint8_t *dst_base, size_t dst_cap,
                               uint64_t *dst_offsets, int *statuses, uint64_t span, zb200_index **indexes);
int zb200_compress_batch_device_index(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                      int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                      size_t dst_cap, uint64_t *dst_offsets, int *statuses, uint64_t span,
                                      zb200_index **indexes);
int zb200_compress_stream_begin_index(zb200_ctx *ctx, int level, int data_format, int fname_len, uint64_t span,
                                      zb200_compress_stream **out);
int zb200_compress_stream_index(zb200_compress_stream *st, zb200_index **out);

/* ---- compression strategies: zlib's `strategy` (deflateInit2, zlib.compressobj) ----
 * The values are zlib's, so Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE and Z_FIXED pass straight through; any other value
 * fails with ZB200_ERR_ARG (and leaves statuses alone, as an invalid level does).  A strategy changes the compressed
 * size, never what the member decodes to: every member is an ordinary stream for any inflater.  Strategy 0 is
 * exactly the calls without _strategy.  The parse is chosen in zlib's order:
 *  - level 0: stored blocks, whatever the strategy;
 *  - level -2, or HUFFMAN_ONLY at any other level: literals only (level -2's bytes);
 *  - RLE at levels -1 and 1..9: a run-length parse, the same bytes at every level.  Each chunk is cut into 4 KiB
 *    pieces; walking left to right, position p (not its chunk's first byte) starts a match of distance 1 when the
 *    byte before it repeats at p, p + 1 and p + 2 inside p's piece, as long as the run goes on (at most 258 and
 *    never past the piece end); otherwise p is a literal.  That is zlib's deflate_rle with no history across a
 *    64 KiB chunk start and no match across a piece end.  There is no history, so a sync and a full flush of a
 *    stream write the same bytes;
 *  - FILTERED at levels -1 and 2..9: the level's parse, with every match shorter than 6 taken as no match before
 *    the one-step lazy rule (zlib deflate_slow's match_length <= 5 rule).  Level 1 ignores it, as zlib's fast
 *    levels do;
 *  - DEFAULT and FIXED: the level's parse.
 * Each chunk's block is the smallest of stored, fixed and dynamic, except under FIXED: the smaller of stored and
 * fixed, never dynamic.  Framing, chunking and the zlib header (78 01 at window 15) do not change, and zb200_compress_bound covers
 * every strategy.  Not combined with dictionaries, compress-time indexes, zb200_compress_batch_h2d or multi-GPU.
 * The _strategy calls take the arguments of the calls without it, plus `strategy` after `level`. */
enum {
  ZB200_STRATEGY_DEFAULT = 0,
  ZB200_STRATEGY_FILTERED = 1,
  ZB200_STRATEGY_HUFFMAN_ONLY = 2,
  ZB200_STRATEGY_RLE = 3,
  ZB200_STRATEGY_FIXED = 4
};
int zb200_compress_batch_strategy(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                  int level, int strategy, int data_format, const uint8_t *fname_lens,
                                  uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_batch_device_strategy(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                         int level, int strategy, int data_format, const uint8_t *fname_lens,
                                         uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_stream_begin_strategy(zb200_ctx *ctx, int level, int strategy, int data_format, int fname_len,
                                         zb200_compress_stream **out);

/* ---- window size: zlib's `windowBits` (deflateInit2, the magnitude of zlib.compressobj's wbits) ----
 * window_bits n in 9..15: no match of any member reaches more than 2^n bytes back, the window RFC 1950 states
 * through CINFO and the one zlib's inflater with wbits = n accepts (zlib's own deflater stops at 2^n - 262; a
 * decoder needs no such margin).  n = 8 is accepted for the zlib format only and means 9, as in zlib; any other n
 * fails with ZB200_ERR_ARG and leaves statuses alone.
 *  - zlib format: CMF = (n - 8) << 4 | 8, FLEVEL 0, FCHECK recomputed (78 01 at n = 15).  gzip and raw DEFLATE have
 *    no window field: only the parse changes;
 *  - n = 15 is exactly the calls without _window, for every level, strategy and format;
 *  - levels 0 and -2, HUFFMAN_ONLY and RLE make no match beyond distance 1 and are unaffected (their zlib header
 *    still states n).  Level 1's matches reach at most 6 KiB back (a 4 KiB piece and its 2 KiB pre-seed), so it
 *    changes only for n <= 12.  Levels -1 and 2..9, FILTERED included, change for every n < 15: a preceding 8 KiB
 *    segment j (0 = nearest) is looked up only when 8192 j < 2^n;
 *  - a stream keeps its window for its whole life: sync flushes, full flushes and the history carried across
 *    writes all respect it.
 * zb200_compress_bound and zb200_compress_stream_bound cover every window.  Not combined with dictionaries,
 * compress-time indexes, zb200_compress_batch_h2d or multi-GPU.  The _window calls take the arguments of the
 * _strategy calls, plus `window_bits` after `strategy`. */
int zb200_compress_batch_window(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int level, int strategy, int window_bits, int data_format, const uint8_t *fname_lens,
                                uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_batch_device_window(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                       int level, int strategy, int window_bits, int data_format,
                                       const uint8_t *fname_lens, uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets,
                                       int *statuses);
int zb200_compress_stream_begin_window(zb200_ctx *ctx, int level, int strategy, int window_bits, int data_format,
                                       int fname_len, zb200_compress_stream **out);

/* ---- optimal parse: the smallest members this library writes (DESIGN.md sections 4 and 5, "k_opt") ----
 * Each 64 KiB chunk is parsed by a shortest path over its candidate matches under integer bit costs, in two cost
 * rounds (fixed-code costs, then the code lengths of the first round's histogram), instead of level 9's lazy
 * matching.  The members are valid gzip / zlib / raw DEFLATE members in the layout of the other calls: one block per
 * 64 KiB chunk, the smallest of stored, fixed and dynamic, chunks joined by empty stored blocks, the zlib header of
 * the _window calls (FLEVEL 0).  zb200_compress_bound and zb200_compress_stream_bound bound them.
 *  - history as at the LZ levels: a chunk sees up to min(32 KiB, 2^window_bits) of the member's earlier bytes; a
 *    stream's sync flush keeps the history, a full flush drops it.  Matches are 4..258 bytes, at most 2^window_bits
 *    back, and none crosses the end of its 8 KiB sub-chunk;
 *  - a member's bytes depend on its input, window_bits, the format and the FNAME length alone (and for a stream on
 *    its flush offsets and modes, not on how the input was split into writes; a stream writes the one-shot member);
 *  - an invalid window_bits fails with ZB200_ERR_ARG and leaves statuses alone.  There is no dictionary,
 *    compress-time index, zb200_compress_batch_h2d or multi-GPU form.
 * The calls take the arguments of the _window calls without `level` and `strategy`; the stream form is driven by the
 * zb200_compress_stream_write / _flush / _finish / _free calls. */
int zb200_compress_batch_optimal(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int window_bits, int data_format, const uint8_t *fname_lens, uint8_t *dst_base,
                                 size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_batch_device_optimal(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                        int window_bits, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                        size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_stream_begin_optimal(zb200_ctx *ctx, int window_bits, int data_format, int fname_len,
                                        zb200_compress_stream **out);

/* ---- rsyncable compression: content-defined chunk starts (DESIGN.md sections 4 and 5, "Rsyncable") ----
 * The _rsyncable calls write one ordinary gzip / zlib / raw DEFLATE member per input, in the layout of the other
 * calls (one block per chunk, chunks joined by empty stored blocks), but a member's chunks start where its content
 * says, not every 64 KiB.  An edit then changes only the compressed bytes near it: the chunks before it keep their
 * bytes, and so do the chunks from the first cut at which the two inputs agree again, as with gzip --rsyncable.
 * The rule, for member bytes m[0..L), is a format promise (it does not change):
 *  - G[b], b = 0..255, is the (b + 1)-th output of splitmix64 started from state 0: each step adds
 *    0x9E3779B97F4A7C15 to the state, then z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27;
 *    z *= 0x94D049BB133111EB; z ^= z >> 31;
 *  - h(0) = 0 and h(p) = 2 h(p - 1) + G[m[p - 1]] mod 2^64 (so h(p) depends on the 64 bytes before p alone);
 *  - p is a candidate if 0 < p < L and h(p) >> 48 == 0;
 *  - a candidate p is an accepted cut if p >= 16384 (MIN) and no other candidate lies in (p - MIN, p);
 *  - each consecutive pair a < b of {0} + cuts + {L} gives the chunk starts a, a + 65536, a + 2 * 65536, ... below
 *    b.  An empty member is one empty chunk at 0.  Without cuts this is the 64 KiB grid of the other calls.
 * So a member of L bytes has at most zb200_rsyncable_chunks_bound(L) = ceil(L / 65536) + floor(L / 16384) chunks
 * (1 for L = 0).  At levels -1 and 2..9 a chunk sees up to 32 KiB of the member in front of its start as history.
 * A member's bytes depend on its input, level, format and FNAME length alone.  zb200_compress_bound can be too small
 * for these members; zb200_compress_bound_rsyncable bounds them.  gzip headers are byte-stable only with fixed
 * fname_lens (compress() in the language bindings draws the FNAME length at random), or in the zlib and raw formats.
 * The host-buffer call copies the whole batch in before it compresses (the map needs every byte first), so it does
 * not overlap copy-in with compression.  There is no stream, dictionary, strategy, window size, compress-time index,
 * optimal-parse, zb200_compress_batch_h2d or multi-GPU form.  The compress calls take the arguments of
 * zb200_compress_batch / zb200_compress_batch_device. */
int zb200_compress_batch_rsyncable(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                   int level, int data_format, const uint8_t *fname_lens, uint8_t *dst_base,
                                   size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_compress_batch_device_rsyncable(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                          int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                          size_t dst_cap, uint64_t *dst_offsets, int *statuses);
size_t zb200_compress_bound_rsyncable(size_t len, int data_format);
size_t zb200_rsyncable_chunks_bound(size_t len);
/* The chunk map the _rsyncable calls compress by (the same code path), for callers that index or deduplicate by
 * chunk: counts[i] receives member i's chunk count, and starts its chunk starts (positions in the member, ascending,
 * the first 0), member after member with nothing between.  starts_cap is the room in starts (entries); the sum of
 * zb200_rsyncable_chunks_bound over the members always suffices.  ZB200_ERR_DST_TOO_SMALL, with counts filled, when
 * the starts do not fit. */
int zb200_rsyncable_chunks(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           uint64_t *counts, uint64_t *starts, size_t starts_cap);

/* ---- device-resident variants (pointers prefixed d_ are device memory on ctx's device;
 * offsets / statuses / sizes stay host arrays).  Used when the data already lives in HBM
 * (bench.py's `value`) and by the multi-GPU sharded path.  The call returns after the
 * work has completed on the ctx stream. ---- */
int zb200_compress_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                int level, int data_format, const uint8_t *fname_lens,
                                uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
/* host inputs -> members left in DEVICE memory (H2D pipelined with the kernels).  The sharded
 * multi-GPU path uses it: compress, exchange the sizes, then copy each shard to its place. */
int zb200_compress_batch_h2d(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                             int level, int data_format, const uint8_t *fname_lens,
                             uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
/* device -> host copy on the ctx stream (returns when it has landed): the second half of the sharded
 * path, once the size exchange has said where a shard goes in the concatenated host stream */
int zb200_download(zb200_ctx *ctx, const uint8_t *d_src, uint8_t *h_dst, size_t bytes);
int zb200_uncompress_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                  int data_format, uint8_t *d_dst, const uint64_t *dst_offsets,
                                  uint64_t *dst_lens, int *statuses);
int zb200_uncompress_sizes_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                  int data_format, uint64_t *sizes, int *statuses);
int zb200_checksum_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                int kind, uint32_t *out);

/* ---- host memory ----
 * The host-buffer calls overlap their copies with the kernels only for page-locked memory.  A caller
 * that reuses a buffer (a Nim string it keeps, an mmap) can page-lock it once with these; buffers that
 * are not page-locked are staged through an internal pinned ring instead (slower than PCIe). */
int zb200_host_register(void *ptr, size_t bytes);
int zb200_host_unregister(void *ptr);

/* ---- several GPUs behind one call (SURVEY 8e at the boundary) ----
 * Members shard by contiguous index range, balanced by bytes; one host thread drives each device through its
 * own ctx; there is no data-path collective.  compress: every shard is compressed on its device, the per-shard
 * sizes are gathered, and each shard's bytes are copied to their place in ONE concatenated host stream
 * (dst_offsets are global).  The multi-process form (one rank per GPU, NCCL all_gather of the sizes) is
 * zippy_b200/sharding.py; this is the same path for a caller that is a single process, e.g. a Nim program.
 * devices == NULL or n_devices <= 0: every visible device.  A device may be listed more than once. */
typedef struct zb200_mgpu zb200_mgpu;
int zb200_mgpu_init(const int *devices, int n_devices, zb200_mgpu **out);
void zb200_mgpu_shutdown(zb200_mgpu *m);
int zb200_mgpu_device_count(zb200_mgpu *m);
int zb200_mgpu_compress_batch(zb200_mgpu *m, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                              int level, int data_format, const uint8_t *fname_lens,
                              uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses);
int zb200_mgpu_uncompress_batch(zb200_mgpu *m, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int data_format, uint8_t *dst_base, const uint64_t *dst_offsets,
                                uint64_t *dst_lens, int *statuses);
int zb200_mgpu_checksum_batch(zb200_mgpu *m, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                              int kind, uint32_t *out);

/* ---- instrumentation (bench.py): device time in ms of the kernels of the last batch call,
 * measured with CUDA events on the ctx stream, and how many kernels it launched. ---- */
typedef struct {
  float lz_ms, huff_ms, scan_ms, pack_ms;      /* compress */
  float inflate_ms, verify_ms;                 /* uncompress */
  float checksum_ms;
  float h2d_ms, d2h_ms;                        /* host-buffer variants only */
  uint64_t h2d_bytes, d2h_bytes;
  uint32_t kernel_launches;
  uint32_t n_chunks;
  float plan_ms;                               /* compress: host time from entry to the first kernel launch */
} zb200_timing;
int zb200_last_timing(zb200_ctx *ctx, zb200_timing *out);

#ifdef __cplusplus
}
#endif
#endif
