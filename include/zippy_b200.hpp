// zippy_b200.hpp -- header-only C++ mirror of guzba/zippy's public API over the C ABI
// (include/zippy_b200.h).  The reference is compiled code (Nim); with no Nim toolchain in
// this environment this is the compiled-language host side: same names, defaults, argument
// meaning and error behaviour as src/zippy.nim:11-177, src/zippy/common.nim:1-12,
// src/zippy/crc.nim:53-75, src/zippy/adler32.nim:6-66.  Framing for the single-input calls is
// done HERE, on the host, exactly where zippy.nim does it; the codec core (deflate, inflate,
// crc32, adler32) goes through the four seam entry points.
#pragma once
#include <cstdint>
#include <random>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "zippy_b200.h"

namespace zippy {

struct ZippyError : std::runtime_error {  // common.nim:2
  int code;
  ZippyError(int c, const std::string &msg) : std::runtime_error(msg), code(c) {}
};

enum CompressedDataFormat { dfDetect = 0, dfZlib = 1, dfGzip = 2, dfDeflate = 3 };  // common.nim:4-5
constexpr int NoCompression = 0, BestSpeed = 1, BestCompression = 9, DefaultCompression = -1, HuffmanOnly = -2;
// zlib's compression strategies, with zlib's values (include/zippy_b200.h "compression strategies")
enum Strategy {
  StrategyDefault = ZB200_STRATEGY_DEFAULT,
  StrategyFiltered = ZB200_STRATEGY_FILTERED,
  StrategyHuffmanOnly = ZB200_STRATEGY_HUFFMAN_ONLY,
  StrategyRle = ZB200_STRATEGY_RLE,
  StrategyFixed = ZB200_STRATEGY_FIXED
};

namespace detail {
inline void check(int rc) {
  if (rc != ZB200_OK) throw ZippyError(rc, zb200_strerror(rc));
}
inline zb200_ctx *ctx() {
  thread_local zb200_ctx *c = nullptr;
  if (!c) check(zb200_init(-1, &c));  // throws without a CUDA device: there is no CPU fallback
  return c;
}
inline const uint8_t *u8(const std::string &s) { return reinterpret_cast<const uint8_t *>(s.data()); }
// deflate.nim:207 -- appends the raw stream to dst
inline void deflate(std::string &dst, const uint8_t *src, size_t len, int level) {
  size_t start = dst.size(), n = 0;
  dst.resize(start + zb200_deflate_bound(len));
  check(zb200_deflate(ctx(), src, len, level, reinterpret_cast<uint8_t *>(&dst[start]), dst.size() - start, &n));
  dst.resize(start + n);
}
// inflate.nim:268
inline void inflate(std::string &dst, const uint8_t *src, size_t len, size_t pos) {
  // one decode: the library inflates into its own device memory, reports the size, then copies out
  size_t n = 0;
  check(zb200_decode_begin(ctx(), src, len, ZB200_DF_DEFLATE, pos, &n));
  dst.resize(n);
  uint8_t dummy = 0;
  check(zb200_decode_finish(ctx(), n ? reinterpret_cast<uint8_t *>(&dst[0]) : &dummy, n, &n));
  dst.resize(n);
}
inline uint32_t read32le(const uint8_t *p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
inline uint32_t read32be(const uint8_t *p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
inline void put32be(std::string &dst, uint32_t v) {
  for (int s = 24; s >= 0; s -= 8) dst.push_back((char)((v >> s) & 255));
}
// the raw stream of src against a preset dictionary (appended to dst): zb200_compress_batch_dict on one input
inline void deflateDict(std::string &dst, const uint8_t *src, size_t len, int level, const std::string &dict) {
  const uint64_t offs[2] = {0, len};
  uint64_t out_offs[2] = {0, 0};
  int st = 0;
  size_t start = dst.size();
  dst.resize(start + zb200_deflate_bound(len) + 64);
  uint8_t dummy = 0;
  check(zb200_compress_batch_dict(ctx(), len ? src : &dummy, offs, 1, level, ZB200_DF_DEFLATE, u8(dict), dict.size(),
                                  reinterpret_cast<uint8_t *>(&dst[start]), dst.size() - start, out_offs, &st));
  dst.resize(start + out_offs[1]);
}
// a raw stream decoded against a preset dictionary: zb200_decode_begin_dict + zb200_decode_finish
inline void inflateDict(std::string &dst, const uint8_t *src, size_t len, const std::string &dict) {
  size_t n = 0;
  uint8_t dummy = 0;
  check(zb200_decode_begin_dict(ctx(), len ? src : &dummy, len, ZB200_DF_DEFLATE, u8(dict), dict.size(), &n));
  dst.resize(n);
  check(zb200_decode_finish(ctx(), n ? reinterpret_cast<uint8_t *>(&dst[0]) : &dummy, n, &n));
  dst.resize(n);
}
}  // namespace detail

inline uint32_t crc32(const void *src, size_t len) {  // crc.nim:53
  uint32_t v = 0;
  detail::check(zb200_crc32(detail::ctx(), src, len, &v));
  return v;
}
inline uint32_t crc32(const std::string &s) { return crc32(s.data(), s.size()); }
inline uint32_t adler32(const void *src, size_t len) {  // adler32.nim:6
  uint32_t v = 0;
  detail::check(zb200_adler32(detail::ctx(), src, len, &v));
  return v;
}
inline uint32_t adler32(const std::string &s) { return adler32(s.data(), s.size()); }

// zippy.nim:11-84
inline std::string compress(const void *srcp, size_t len, int level = DefaultCompression,
                            CompressedDataFormat dataFormat = dfGzip) {
  const uint8_t *src = static_cast<const uint8_t *>(srcp);
  std::string result;
  switch (dataFormat) {
    case dfGzip: {
      result.assign({31, (char)139, 8, 1 << 3, 0, 0, 0, 0, 0, 0});
      std::random_device rd;  // zippy.nim:28-42: 0..25 letters against BREACH-style length probing
      int k = (int)(rd() % 26);
      for (int i = 0; i < k; i++) result.push_back((char)(97 + i));
      result.push_back('\0');
      detail::deflate(result, src, len, level);
      uint32_t c = crc32(src, len), isz = (uint32_t)len;
      for (int s = 0; s < 32; s += 8) result.push_back((char)((c >> s) & 255));
      for (int s = 0; s < 32; s += 8) result.push_back((char)((isz >> s) & 255));
      return result;
    }
    case dfZlib: {
      result.assign({0x78, 0x01});
      detail::deflate(result, src, len, level);
      uint32_t a = adler32(src, len);
      for (int s = 24; s >= 0; s -= 8) result.push_back((char)((a >> s) & 255));
      return result;
    }
    case dfDeflate:
      detail::deflate(result, src, len, level);
      return result;
    default:
      throw ZippyError(ZB200_ERR_INVALID_FORMAT, "Invalid data format dfDetect");
  }
}
inline std::string compress(const std::string &src, int level = DefaultCompression,
                            CompressedDataFormat dataFormat = dfGzip) {
  return compress(src.data(), src.size(), level, dataFormat);
}
// With a preset dictionary (zlib's zdict; include/zippy_b200.h "preset dictionaries"): zlib members start 78 20 and
// the DICTID (the Adler-32 of the whole dictionary), raw members carry nothing, gzip is refused.  An empty dictionary
// is the call without one.
inline std::string compress(const void *srcp, size_t len, int level, CompressedDataFormat dataFormat,
                            const std::string &dictionary) {
  if (dictionary.empty()) return compress(srcp, len, level, dataFormat);
  if (level < -2 || level > 9) throw ZippyError(ZB200_ERR_INVALID_LEVEL, "Invalid compression level");
  if (dataFormat != dfZlib && dataFormat != dfDeflate) throw ZippyError(ZB200_ERR_INVALID_FORMAT, "Invalid data format");
  const uint8_t *src = static_cast<const uint8_t *>(srcp);
  std::string result;
  if (dataFormat == dfZlib) {
    result.assign({0x78, 0x20});
    detail::put32be(result, adler32(dictionary));
  }
  detail::deflateDict(result, src, len, level, dictionary);
  if (dataFormat == dfZlib) detail::put32be(result, adler32(src, len));
  return result;
}
inline std::string compress(const std::string &src, int level, CompressedDataFormat dataFormat,
                            const std::string &dictionary) {
  return compress(src.data(), src.size(), level, dataFormat, dictionary);
}

// Under a compression strategy: one member of zb200_compress_batch_strategy (gzip draws its FNAME length at
// random, as compress() does).  StrategyDefault writes compress()'s bytes.
inline std::string compress(const void *srcp, size_t len, int level, CompressedDataFormat dataFormat, Strategy strategy) {
  const uint64_t offs[2] = {0, len};
  uint64_t out_offs[2] = {0, 0};
  int st = 0;
  const uint8_t fl = dataFormat == dfGzip ? (uint8_t)(std::random_device()() % 26) : 0;
  std::string result(zb200_compress_bound(len, dataFormat) + 64, '\0');
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_strategy(detail::ctx(), len ? static_cast<const uint8_t *>(srcp) : &dummy, offs, 1,
                                              level, strategy, dataFormat, &fl, reinterpret_cast<uint8_t *>(&result[0]),
                                              result.size(), out_offs, &st));
  result.resize(out_offs[1]);
  return result;
}
inline std::string compress(const std::string &src, int level, CompressedDataFormat dataFormat, Strategy strategy) {
  return compress(src.data(), src.size(), level, dataFormat, strategy);
}

// With zlib's window size (windowBits 9..15; 8 for dfZlib means 9): one member of zb200_compress_batch_window, no
// match reaching more than 2^windowBits back.  windowBits 15 writes the overload above's bytes.
inline std::string compress(const void *srcp, size_t len, int level, CompressedDataFormat dataFormat, Strategy strategy,
                            int windowBits) {
  const uint64_t offs[2] = {0, len};
  uint64_t out_offs[2] = {0, 0};
  int st = 0;
  const uint8_t fl = dataFormat == dfGzip ? (uint8_t)(std::random_device()() % 26) : 0;
  std::string result(zb200_compress_bound(len, dataFormat) + 64, '\0');
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_window(detail::ctx(), len ? static_cast<const uint8_t *>(srcp) : &dummy, offs, 1,
                                            level, strategy, windowBits, dataFormat, &fl,
                                            reinterpret_cast<uint8_t *>(&result[0]), result.size(), out_offs, &st));
  result.resize(out_offs[1]);
  return result;
}
inline std::string compress(const std::string &src, int level, CompressedDataFormat dataFormat, Strategy strategy,
                            int windowBits) {
  return compress(src.data(), src.size(), level, dataFormat, strategy, windowBits);
}

// The optimal parse (zb200_compress_batch_optimal): smaller members than level 9, with zlib's window size
// (windowBits 9..15; 8 for dfZlib means 9).  No strategy, dictionary or index.
inline std::string compressOptimal(const void *srcp, size_t len, CompressedDataFormat dataFormat, int windowBits = 15) {
  const uint64_t offs[2] = {0, len};
  uint64_t out_offs[2] = {0, 0};
  int st = 0;
  const uint8_t fl = dataFormat == dfGzip ? (uint8_t)(std::random_device()() % 26) : 0;
  std::string result(zb200_compress_bound(len, dataFormat) + 64, '\0');
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_optimal(detail::ctx(), len ? static_cast<const uint8_t *>(srcp) : &dummy, offs, 1,
                                             windowBits, dataFormat, &fl, reinterpret_cast<uint8_t *>(&result[0]),
                                             result.size(), out_offs, &st));
  result.resize(out_offs[1]);
  return result;
}
inline std::string compressOptimal(const std::string &src, CompressedDataFormat dataFormat, int windowBits = 15) {
  return compressOptimal(src.data(), src.size(), dataFormat, windowBits);
}

// Rsyncable compression (zb200_compress_batch_rsyncable): chunk starts taken from the content, so an edit changes
// only the compressed bytes near it.  Any level and format; a gzip member's FNAME length is drawn at random, as
// compress() does (fnameLen >= 0 fixes it, for byte-stable gzip output).
inline std::string compressRsyncable(const void *srcp, size_t len, int level = DefaultCompression,
                                     CompressedDataFormat dataFormat = dfGzip, int fnameLen = -1) {
  const uint64_t offs[2] = {0, len};
  uint64_t out_offs[2] = {0, 0};
  int st = 0;
  const uint8_t fl = fnameLen >= 0 ? (uint8_t)fnameLen
                                   : dataFormat == dfGzip ? (uint8_t)(std::random_device()() % 26) : 0;
  std::string result(zb200_compress_bound_rsyncable(len, dataFormat) + 64, '\0');
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_rsyncable(detail::ctx(), len ? static_cast<const uint8_t *>(srcp) : &dummy, offs,
                                               1, level, dataFormat, &fl, reinterpret_cast<uint8_t *>(&result[0]),
                                               result.size(), out_offs, &st));
  result.resize(out_offs[1]);
  return result;
}
inline std::string compressRsyncable(const std::string &src, int level = DefaultCompression,
                                     CompressedDataFormat dataFormat = dfGzip, int fnameLen = -1) {
  return compressRsyncable(src.data(), src.size(), level, dataFormat, fnameLen);
}
// one member per input, one launch sequence; fnameLens: one gzip FNAME length (0..25) per input, or empty for none
inline std::vector<std::string> compressRsyncableBatch(const std::vector<std::string> &srcs, int level = DefaultCompression,
                                                      CompressedDataFormat dataFormat = dfGzip,
                                                      const std::vector<uint8_t> &fnameLens = {}) {
  std::vector<uint64_t> offs(srcs.size() + 1, 0), out_offs(srcs.size() + 1, 0);
  std::string all;
  size_t cap = 64;
  for (size_t i = 0; i < srcs.size(); i++) {
    all += srcs[i];
    offs[i + 1] = all.size();
    cap += zb200_compress_bound_rsyncable(srcs[i].size(), dataFormat) + 64;
  }
  std::vector<int> st(srcs.size() + 1, 0);
  std::string out(cap, '\0');
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_rsyncable(
      detail::ctx(), all.empty() ? &dummy : reinterpret_cast<const uint8_t *>(all.data()), offs.data(), srcs.size(),
      level, dataFormat, fnameLens.empty() ? nullptr : fnameLens.data(), reinterpret_cast<uint8_t *>(&out[0]),
      out.size(), out_offs.data(), st.data()));
  std::vector<std::string> result;
  for (size_t i = 0; i < srcs.size(); i++) result.push_back(out.substr(out_offs[i], out_offs[i + 1] - out_offs[i]));
  return result;
}

// gzip.nim:3-88
inline void uncompressGzip(std::string &dst, const uint8_t *src, size_t len) {
  auto fail = [] { throw ZippyError(ZB200_ERR_UNCOMPRESS, "Invalid buffer, unable to uncompress"); };
  if (len < 18) fail();
  if (src[0] != 31 || src[1] != 139) throw ZippyError(ZB200_ERR_GZIP_ID, "Failed gzip identification values check");
  if (src[2] != 8) throw ZippyError(ZB200_ERR_METHOD, "Unsupported compression method");
  uint8_t flg = src[3];
  if (flg & 0xe0) throw ZippyError(ZB200_ERR_GZIP_RESERVED, "Reserved flag bits set");
  if (flg & 4) throw ZippyError(ZB200_ERR_GZIP_FLAGS, "Currently unsupported flags are set");
  size_t pos = 10;
  for (int pass = 0; pass < 2; pass++)
    if ((pass == 0 && (flg & 8)) || (pass == 1 && (flg & 16))) {
      while (pos < len && src[pos] != 0) pos++;
      if (pos >= len) fail();
      pos++;
    }
  if (flg & 2) {
    if (pos + 2 >= len) fail();
    pos += 2;
  }
  if (pos + 8 >= len) fail();
  uint32_t checksum = detail::read32le(src + len - 8), isize = detail::read32le(src + len - 4);
  detail::inflate(dst, src, len, pos);
  if (checksum != crc32(dst)) throw ZippyError(ZB200_ERR_CHECKSUM, "Checksum verification failed");
  if (isize != (uint32_t)dst.size()) throw ZippyError(ZB200_ERR_SIZE, "Size verification failed");
}

// zippy.nim:100-165
inline std::string uncompress(const void *srcp, size_t len, CompressedDataFormat dataFormat = dfDetect) {
  const uint8_t *src = static_cast<const uint8_t *>(srcp);
  std::string result;
  switch (dataFormat) {
    case dfDetect:
      if (len > 18 && src[0] == 31 && src[1] == 139 && src[2] == 8 && (src[3] & 0xe0) == 0)
        return uncompress(src, len, dfGzip);
      if (len > 6 && (src[0] & 0x0f) == 8 && (src[0] >> 4) <= 7 && (((uint32_t)src[0] * 256u) + src[1]) % 31u == 0)
        return uncompress(src, len, dfZlib);
      throw ZippyError(ZB200_ERR_DETECT, "Unable to detect compressed data format");
    case dfGzip:
      uncompressGzip(result, src, len);
      return result;
    case dfZlib: {
      if (len < 6) throw ZippyError(ZB200_ERR_UNCOMPRESS, "Invalid buffer, unable to uncompress");
      uint8_t cmf = src[0], flg = src[1];
      if ((cmf & 0x0f) != 8) throw ZippyError(ZB200_ERR_METHOD, "Unsupported compression method");
      if ((cmf >> 4) > 7) throw ZippyError(ZB200_ERR_CINFO, "Invalid compression info");
      if ((((uint32_t)cmf * 256u) + flg) % 31u != 0) throw ZippyError(ZB200_ERR_HEADER, "Invalid header");
      if (flg & 0x20) throw ZippyError(ZB200_ERR_FDICT, "Preset dictionary is not yet supported");
      detail::inflate(result, src, len, 2);
      uint32_t checksum = ((uint32_t)src[len - 4] << 24) | ((uint32_t)src[len - 3] << 16) |
                          ((uint32_t)src[len - 2] << 8) | src[len - 1];
      if (checksum != adler32(result)) throw ZippyError(ZB200_ERR_CHECKSUM, "Checksum verification failed");
      return result;
    }
    case dfDeflate:
      detail::inflate(result, src, len, 0);
      return result;
  }
  throw ZippyError(ZB200_ERR_INVALID_FORMAT, "Invalid data format");
}
inline std::string uncompress(const std::string &src, CompressedDataFormat dataFormat = dfDetect) {
  return uncompress(src.data(), src.size(), dataFormat);
}
// With a preset dictionary: raw members, and zlib members with FDICT, decode against it (a DICTID that is not the
// dictionary's: ZB200_ERR_DICTIONARY); gzip members and zlib members without FDICT ignore it.  An empty dictionary
// is the call without one.
inline std::string uncompress(const void *srcp, size_t len, CompressedDataFormat dataFormat,
                              const std::string &dictionary) {
  if (dictionary.empty()) return uncompress(srcp, len, dataFormat);
  const uint8_t *src = static_cast<const uint8_t *>(srcp);
  std::string result;
  switch (dataFormat) {
    case dfDetect:
      if (len > 18 && src[0] == 31 && src[1] == 139 && src[2] == 8 && (src[3] & 0xe0) == 0)
        return uncompress(src, len, dfGzip);
      if (len > 6 && (src[0] & 0x0f) == 8 && (src[0] >> 4) <= 7 && (((uint32_t)src[0] * 256u) + src[1]) % 31u == 0)
        return uncompress(src, len, dfZlib, dictionary);
      throw ZippyError(ZB200_ERR_DETECT, "Unable to detect compressed data format");
    case dfGzip:
      return uncompress(src, len, dfGzip);
    case dfZlib: {
      if (len < 6 || !(src[1] & 0x20)) return uncompress(src, len, dfZlib);
      uint8_t cmf = src[0], flg = src[1];
      if ((cmf & 0x0f) != 8) throw ZippyError(ZB200_ERR_METHOD, "Unsupported compression method");
      if ((cmf >> 4) > 7) throw ZippyError(ZB200_ERR_CINFO, "Invalid compression info");
      if ((((uint32_t)cmf * 256u) + flg) % 31u != 0) throw ZippyError(ZB200_ERR_HEADER, "Invalid header");
      if (len < 10) throw ZippyError(ZB200_ERR_UNCOMPRESS, "Invalid buffer, unable to uncompress");
      if (detail::read32be(src + 2) != adler32(dictionary))
        throw ZippyError(ZB200_ERR_DICTIONARY, zb200_strerror(ZB200_ERR_DICTIONARY));
      detail::inflateDict(result, src + 6, len - 6, dictionary);
      if (detail::read32be(src + len - 4) != adler32(result))
        throw ZippyError(ZB200_ERR_CHECKSUM, "Checksum verification failed");
      return result;
    }
    case dfDeflate:
      detail::inflateDict(result, src, len, dictionary);
      return result;
  }
  throw ZippyError(ZB200_ERR_INVALID_FORMAT, "Invalid data format");
}
inline std::string uncompress(const std::string &src, CompressedDataFormat dataFormat, const std::string &dictionary) {
  return uncompress(src.data(), src.size(), dataFormat, dictionary);
}

// One GPU launch sequence for many inputs (no reference counterpart; cf. the loop over entries
// in ziparchives.nim:505-540).
inline std::vector<std::string> compressBatch(const std::vector<std::string> &items, int level = DefaultCompression,
                                              CompressedDataFormat dataFormat = dfGzip) {
  std::string base;
  std::vector<uint64_t> offs(items.size() + 1, 0), out_offs(items.size() + 1, 0);
  size_t bound = 64;
  for (size_t i = 0; i < items.size(); i++) {
    base += items[i];
    offs[i + 1] = base.size();
    bound += zb200_compress_bound(items[i].size(), dataFormat) + 64;
  }
  std::string out(bound, '\0');
  std::vector<int> st(items.size() + 1, 0);
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch(detail::ctx(), items.empty() ? &dummy : detail::u8(base), offs.data(), items.size(),
                                     level, dataFormat, nullptr, reinterpret_cast<uint8_t *>(&out[0]), out.size(),
                                     out_offs.data(), st.data()));
  std::vector<std::string> res;
  for (size_t i = 0; i < items.size(); i++) res.emplace_back(out.substr(out_offs[i], out_offs[i + 1] - out_offs[i]));
  return res;
}

namespace detail {
// a dictionary table (include/zippy_b200.h "per-member preset dictionaries") as base + k + 1 offsets
inline std::string packDicts(const std::vector<std::string> &dicts, std::vector<uint64_t> &offs) {
  std::string base;
  offs.assign(dicts.size() + 1, 0);
  for (size_t j = 0; j < dicts.size(); j++) {
    base += dicts[j];
    offs[j + 1] = base.size();
  }
  return base;
}
}  // namespace detail

// Per-member preset dictionaries at zlib's window size (zb200_compress_batch_dicts): item i is compressed against
// dicts[dictOf[i]], or without a dictionary for dictOf[i] == -1; windowBits 9..15 (8 for dfZlib means 9).
inline std::vector<std::string> compressBatch(const std::vector<std::string> &items, int level,
                                              CompressedDataFormat dataFormat, int windowBits,
                                              const std::vector<std::string> &dicts, const std::vector<int32_t> &dictOf) {
  if (dictOf.size() != items.size()) throw ZippyError(ZB200_ERR_ARG, "dictOf needs one entry per item");
  std::string base;
  std::vector<uint64_t> offs(items.size() + 1, 0), out_offs(items.size() + 1, 0), doffs;
  size_t bound = 64;
  for (size_t i = 0; i < items.size(); i++) {
    base += items[i];
    offs[i + 1] = base.size();
    bound += zb200_compress_bound(items[i].size(), dataFormat) + 4 + 64;
  }
  const std::string dbase = detail::packDicts(dicts, doffs);
  std::string out(bound, '\0');
  std::vector<int> st(items.size() + 1, 0);
  uint8_t dummy = 0;
  detail::check(zb200_compress_batch_dicts(detail::ctx(), items.empty() ? &dummy : detail::u8(base), offs.data(),
                                           items.size(), level, dataFormat, windowBits,
                                           dbase.empty() ? &dummy : detail::u8(dbase), doffs.data(), dicts.size(),
                                           dictOf.data(), reinterpret_cast<uint8_t *>(&out[0]), out.size(),
                                           out_offs.data(), st.data()));
  std::vector<std::string> res;
  for (size_t i = 0; i < items.size(); i++) res.emplace_back(out.substr(out_offs[i], out_offs[i + 1] - out_offs[i]));
  return res;
}

// Members decoded against per-member preset dictionaries (zb200_uncompress_sizes_dicts, then
// zb200_uncompress_batch_dicts): member i against dicts[dictOf[i]], or none for -1.  A member that does not decode
// throws its status.
inline std::vector<std::string> uncompressBatch(const std::vector<std::string> &members, CompressedDataFormat dataFormat,
                                                const std::vector<std::string> &dicts,
                                                const std::vector<int32_t> &dictOf) {
  if (dictOf.size() != members.size()) throw ZippyError(ZB200_ERR_ARG, "dictOf needs one entry per member");
  const size_t n = members.size();
  std::string base;
  std::vector<uint64_t> offs(n + 1, 0), doffs, sizes(n + 1, 0), dst_offs(n + 1, 0), lens(n + 1, 0);
  for (size_t i = 0; i < n; i++) {
    base += members[i];
    offs[i + 1] = base.size();
  }
  const std::string dbase = detail::packDicts(dicts, doffs);
  std::vector<int> st(n + 1, 0);
  uint8_t dummy = 0;
  const uint8_t *src = n ? detail::u8(base) : &dummy, *db = dbase.empty() ? &dummy : detail::u8(dbase);
  detail::check(zb200_uncompress_sizes_dicts(detail::ctx(), src, offs.data(), n, dataFormat, db, doffs.data(),
                                             dicts.size(), dictOf.data(), sizes.data(), st.data()));
  for (size_t i = 0; i < n; i++) {
    detail::check(st[i]);
    dst_offs[i + 1] = dst_offs[i] + sizes[i];
  }
  std::string out(dst_offs[n] + 64, '\0');
  detail::check(zb200_uncompress_batch_dicts(detail::ctx(), src, offs.data(), n, dataFormat, db, doffs.data(),
                                             dicts.size(), dictOf.data(), reinterpret_cast<uint8_t *>(&out[0]),
                                             dst_offs.data(), lens.data(), st.data()));
  std::vector<std::string> res;
  for (size_t i = 0; i < n; i++) {
    detail::check(st[i]);
    res.emplace_back(out.substr(dst_offs[i], lens[i]));
  }
  return res;
}

// One member compressed from input that arrives piece by piece (zb200_compress_stream_*, no reference
// counterpart): what write() and finish() return, concatenated, is the member compressBatch writes for the whole
// input with the same FNAME length.  Small writes are gathered and return "".  fnameLen < 0 with gzip draws the
// FNAME length at random, as compress() does; ctx nullptr is this thread's default context.
class Index;
class CompressStream {
 public:
  explicit CompressStream(int level = DefaultCompression, CompressedDataFormat dataFormat = dfGzip, int fnameLen = -1,
                          zb200_ctx *ctx = nullptr) {
    if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
    detail::check(zb200_compress_stream_begin(ctx ? ctx : detail::ctx(), level, dataFormat, fnameLen, &st_));
  }
  // with a preset dictionary (zlib / raw; no FNAME): zb200_compress_stream_begin_dict
  CompressStream(int level, CompressedDataFormat dataFormat, const std::string &dictionary, zb200_ctx *ctx = nullptr) {
    detail::check(zb200_compress_stream_begin_dict(ctx ? ctx : detail::ctx(), level, dataFormat, detail::u8(dictionary),
                                                   dictionary.size(), &st_));
  }
  // under a compression strategy (zb200_compress_stream_begin_strategy)
  CompressStream(int level, CompressedDataFormat dataFormat, Strategy strategy, int fnameLen = -1, zb200_ctx *ctx = nullptr) {
    if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
    detail::check(zb200_compress_stream_begin_strategy(ctx ? ctx : detail::ctx(), level, strategy, dataFormat, fnameLen, &st_));
  }
  // with a window size, kept for the stream's whole life (zb200_compress_stream_begin_window); fnameLen -1 draws it
  // (it has no default: four arguments are the strategy constructor's, with fnameLen)
  CompressStream(int level, CompressedDataFormat dataFormat, Strategy strategy, int windowBits, int fnameLen,
                 zb200_ctx *ctx = nullptr) {
    if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
    detail::check(zb200_compress_stream_begin_window(ctx ? ctx : detail::ctx(), level, strategy, windowBits, dataFormat,
                                                     fnameLen, &st_));
  }
  // the optimal parse (zb200_compress_stream_begin_optimal), selected by the tag CompressStream::Optimal{}
  struct Optimal {};
  CompressStream(Optimal, CompressedDataFormat dataFormat, int windowBits = 15, int fnameLen = -1, zb200_ctx *ctx = nullptr) {
    if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
    detail::check(zb200_compress_stream_begin_optimal(ctx ? ctx : detail::ctx(), windowBits, dataFormat, fnameLen, &st_));
  }
  // that also writes the member's index (zb200_compress_stream_begin_index): index() after finish()
  CompressStream(int level, CompressedDataFormat dataFormat, int fnameLen, uint64_t indexSpan, zb200_ctx *ctx = nullptr)
      : ctx_(ctx ? ctx : detail::ctx()) {
    if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
    detail::check(zb200_compress_stream_begin_index(ctx_, level, dataFormat, fnameLen, indexSpan, &st_));
  }
  ~CompressStream() { zb200_compress_stream_free(st_); }
  CompressStream(const CompressStream &) = delete;
  CompressStream &operator=(const CompressStream &) = delete;

  std::string write(const void *src, size_t len) {
    std::string out(zb200_compress_stream_bound(st_, len), '\0');
    size_t n = 0;
    detail::check(zb200_compress_stream_write(st_, static_cast<const uint8_t *>(src), len,
                                              reinterpret_cast<uint8_t *>(&out[0]), out.size(), &n));
    out.resize(n);
    return out;
  }
  std::string write(const std::string &data) { return write(data.data(), data.size()); }
  // Emit everything written so far (ZB200_SYNC_FLUSH keeps the history, ZB200_FULL_FLUSH drops it): the
  // bytes returned so far decode to the bytes written so far.  "" when nothing was written since the last flush.
  std::string flush(int mode = ZB200_SYNC_FLUSH) {
    std::string out(zb200_compress_stream_bound(st_, 0), '\0');
    size_t n = 0;
    detail::check(zb200_compress_stream_flush(st_, mode, reinterpret_cast<uint8_t *>(&out[0]), out.size(), &n));
    out.resize(n);
    return out;
  }
  std::string finish() {
    std::string out(zb200_compress_stream_bound(st_, 0), '\0');
    size_t n = 0;
    detail::check(zb200_compress_stream_finish(st_, reinterpret_cast<uint8_t *>(&out[0]), out.size(), &n));
    out.resize(n);
    return out;
  }
  Index index() const;  // after finish() on a stream begun with an index span

 private:
  zb200_compress_stream *st_ = nullptr;
  zb200_ctx *ctx_ = nullptr;
};

// One member decoded from compressed input that arrives piece by piece (zb200_decompress_stream_*, no reference
// counterpart): what write() and finish() return, concatenated, is uncompress(whole input, dataFormat); a bad input
// throws the ZippyError uncompress throws.  Small writes are gathered and return "".  ctx nullptr is this thread's
// default context.
class DecompressStream {
 public:
  explicit DecompressStream(CompressedDataFormat dataFormat = dfDetect, zb200_ctx *ctx = nullptr) {
    detail::check(zb200_decompress_stream_begin(ctx ? ctx : detail::ctx(), dataFormat, &st_));
  }
  // with a preset dictionary: zb200_decompress_stream_begin_dict
  DecompressStream(CompressedDataFormat dataFormat, const std::string &dictionary, zb200_ctx *ctx = nullptr) {
    detail::check(zb200_decompress_stream_begin_dict(ctx ? ctx : detail::ctx(), dataFormat, detail::u8(dictionary),
                                                     dictionary.size(), &st_));
  }
  ~DecompressStream() { zb200_decompress_stream_free(st_); }
  DecompressStream(const DecompressStream &) = delete;
  DecompressStream &operator=(const DecompressStream &) = delete;

  std::string write(const void *src, size_t len) {
    size_t avail = 0;
    detail::check(zb200_decompress_stream_write(st_, static_cast<const uint8_t *>(src), len, &avail));
    return take(avail);
  }
  std::string write(const std::string &data) { return write(data.data(), data.size()); }
  // Decode every block that is complete in the input so far, whatever the batching threshold: after a sender's
  // flush, everything it wrote up to the flush.
  std::string drain() {
    size_t avail = 0;
    detail::check(zb200_decompress_stream_drain(st_, &avail));
    return take(avail);
  }
  std::string finish() {
    size_t avail = 0;
    detail::check(zb200_decompress_stream_finish(st_, &avail));
    return take(avail);
  }

 private:
  std::string take(size_t avail) {
    std::string out(avail, '\0');
    size_t n = 0;
    detail::check(zb200_decompress_stream_read(st_, reinterpret_cast<uint8_t *>(&out[0]), out.size(), &n));
    out.resize(n);
    return out;
  }
  zb200_decompress_stream *st_ = nullptr;
};

// Random access into one member (zb200_index_*): build once, then read ranges of its output.
class Index {
 public:
  static Index build(const std::string &data, CompressedDataFormat dataFormat = dfDetect, uint64_t span = 1u << 20,
                     zb200_ctx *ctx = nullptr) {
    Index ix(ctx);
    detail::check(zb200_index_build(ix.ctx_, reinterpret_cast<const uint8_t *>(data.data()), data.size(), dataFormat,
                                    span, &ix.idx_));
    return ix;
  }
  static Index fromBytes(const std::string &buf, zb200_ctx *ctx = nullptr) {
    Index ix(ctx);
    detail::check(zb200_index_import(ix.ctx_, reinterpret_cast<const uint8_t *>(buf.data()), buf.size(), &ix.idx_));
    return ix;
  }
  Index(Index &&o) noexcept : ctx_(o.ctx_), idx_(o.idx_) { o.idx_ = nullptr; }
  Index &operator=(Index &&o) noexcept {
    std::swap(ctx_, o.ctx_);
    std::swap(idx_, o.idx_);
    return *this;
  }
  Index(const Index &) = delete;
  Index &operator=(const Index &) = delete;
  ~Index() { close(); }

  uint64_t size() const { return zb200_index_size(idx_); }
  struct Point {
    uint64_t bit, out;
    uint32_t crc;
    bool window;
  };
  std::vector<Point> points() const {
    const size_t n = zb200_index_points(idx_, nullptr, nullptr, nullptr, nullptr, 0);
    std::vector<uint64_t> b(n), o(n);
    std::vector<uint32_t> c(n);
    std::vector<uint8_t> w(n);
    zb200_index_points(idx_, b.data(), o.data(), c.data(), w.data(), n);
    std::vector<Point> out(n);
    for (size_t i = 0; i < n; i++) out[i] = Point{b[i], o[i], c[i], w[i] != 0};
    return out;
  }
  // ranges [offsets[i], offsets[i] + lengths[i]); statuses[i] == 0 where out[i] holds the bytes
  std::vector<std::string> extractBatch(const std::string &data, const std::vector<uint64_t> &offsets,
                                        const std::vector<uint64_t> &lengths, std::vector<int> &statuses) const {
    if (offsets.size() != lengths.size()) detail::check(ZB200_ERR_ARG);
    const size_t n = offsets.size();
    std::vector<uint64_t> doff(n + 1, 0);
    for (size_t i = 0; i < n; i++) doff[i + 1] = doff[i] + lengths[i];
    std::string buf(doff[n] + 1, '\0');
    statuses.assign(n, 0);
    detail::check(zb200_index_extract_batch(ctx_, idx_, reinterpret_cast<const uint8_t *>(data.data()), data.size(),
                                            offsets.data(), lengths.data(), n, reinterpret_cast<uint8_t *>(&buf[0]),
                                            doff.data(), statuses.data()));
    std::vector<std::string> out(n);
    for (size_t i = 0; i < n; i++)
      if (statuses[i] == 0) out[i] = buf.substr(doff[i], lengths[i]);
    return out;
  }
  std::string extract(const std::string &data, uint64_t offset, uint64_t length) const {
    std::vector<int> st;
    std::vector<std::string> r = extractBatch(data, {offset}, {length}, st);
    detail::check(st[0]);
    return r[0];
  }
  std::string toBytes() const {
    size_t n = 0;
    detail::check(zb200_index_export(ctx_, idx_, nullptr, 0, &n));
    std::string out(n, '\0');
    detail::check(zb200_index_export(ctx_, idx_, reinterpret_cast<uint8_t *>(&out[0]), out.size(), &n));
    out.resize(n);
    return out;
  }
  void close() {
    zb200_index_free(idx_);
    idx_ = nullptr;
  }

 private:
  friend class CompressStream;
  friend std::pair<std::string, Index> compressWithIndex(const std::string &, int, CompressedDataFormat, uint64_t, int,
                                                         zb200_ctx *);
  explicit Index(zb200_ctx *ctx) : ctx_(ctx ? ctx : detail::ctx()) {}
  zb200_ctx *ctx_ = nullptr;
  zb200_index *idx_ = nullptr;
};

inline Index CompressStream::index() const {
  Index ix(ctx_);
  detail::check(zb200_compress_stream_index(st_, &ix.idx_));
  return ix;
}

// compress() that also returns the member's index, the one Index::build(member, dataFormat, span) gives, written
// while compressing (zb200_compress_batch_index).  fnameLen < 0: a random gzip FNAME length, as compress() draws.
inline std::pair<std::string, Index> compressWithIndex(const std::string &src, int level = DefaultCompression,
                                                       CompressedDataFormat dataFormat = dfGzip, uint64_t span = 1u << 20,
                                                       int fnameLen = -1, zb200_ctx *ctx = nullptr) {
  Index ix(ctx);
  if (fnameLen < 0) fnameLen = dataFormat == dfGzip ? (int)(std::random_device()() % 26) : 0;
  const uint8_t fl = (uint8_t)fnameLen;
  const uint64_t offs[2] = {0, src.size()};
  uint64_t doffs[2] = {0, 0};
  int st = 0;
  std::string out(zb200_compress_bound(src.size(), dataFormat) + 64, '\0');
  detail::check(zb200_compress_batch_index(ix.ctx_, detail::u8(src), offs, 1, level, dataFormat, &fl,
                                           reinterpret_cast<uint8_t *>(&out[0]), out.size(), doffs, &st, span, &ix.idx_));
  out.resize(doffs[1]);
  return {std::move(out), std::move(ix)};
}

}  // namespace zippy
