// zb_wrapper.h -- gzip / zlib wrapper validation shared by the device decoder and the host
// (sizing without touching the device, planning of large members): one definition, one behaviour.
#pragma once
#include "zb_common.h"

ZB_HD uint32_t zb_ld_le32(const uint8_t *p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}


// zippy.nim:100-165 + gzip.nim:3-66: resolve the format, validate the wrapper, find the
// payload start and the trailer checksum.  On the device all lanes of a group run this redundantly.
// dict_id: null (no dictionary: FDICT is ZB_ERR_FDICT), or the DICTID (Adler-32) of the caller's non-empty
// dictionary: a zlib member with FDICT then needs 10 bytes and that DICTID, and its payload starts at byte 6.
ZB_HD int zb_parse_wrapper(const uint8_t *src, uint64_t len, int fmt, uint64_t raw_pos,
                                             uint64_t &pos, uint32_t &kind, uint32_t &expect, uint32_t &isize,
                                             const uint32_t *dict_id = nullptr) {
  expect = 0;
  isize = 0;
  if (fmt == ZB_DF_DETECT) {
    if (len > 18 && src[0] == 31 && src[1] == 139 && src[2] == 8 && (src[3] & 0xe0) == 0) fmt = ZB_DF_GZIP;
    else if (len > 6 && (src[0] & 0x0f) == 8 && (src[0] >> 4) <= 7 && (((uint32_t)src[0] * 256u) + src[1]) % 31u == 0)
      fmt = ZB_DF_ZLIB;
    else return ZB_ERR_DETECT;
  }
  kind = (uint32_t)fmt;
  if (fmt == ZB_DF_GZIP) {
    if (len < 18) return ZB_ERR_UNCOMPRESS;
    uint32_t flg = src[3];
    if (src[0] != 31 || src[1] != 139) return ZB_ERR_GZIP_ID;
    if (src[2] != 8) return ZB_ERR_METHOD;
    if (flg & 0xe0) return ZB_ERR_GZIP_RESERVED;
    if (flg & 4) return ZB_ERR_GZIP_FLAGS;
    uint64_t p = 10;
    for (int pass = 0; pass < 2; pass++) {
      if ((pass == 0 && (flg & 8)) || (pass == 1 && (flg & 16))) {
        while (p < len && src[p] != 0) p++;
        if (p >= len) return ZB_ERR_UNCOMPRESS;
        p++;
      }
    }
    if (flg & 2) {
      if (p + 2 >= len) return ZB_ERR_UNCOMPRESS;
      p += 2;
    }
    if (p + 8 >= len) return ZB_ERR_UNCOMPRESS;
    expect = zb_ld_le32(src + len - 8);
    isize = zb_ld_le32(src + len - 4);
    pos = p;
    return ZB_OK;
  }
  if (fmt == ZB_DF_ZLIB) {
    if (len < 6) return ZB_ERR_UNCOMPRESS;
    uint32_t cmf = src[0], flg = src[1];
    if ((cmf & 0x0f) != 8) return ZB_ERR_METHOD;
    if ((cmf >> 4) > 7) return ZB_ERR_CINFO;
    if ((cmf * 256u + flg) % 31u != 0) return ZB_ERR_HEADER;
    pos = 2;
    if (flg & 0x20) {
      if (!dict_id) return ZB_ERR_FDICT;
      if (len < 10) return ZB_ERR_UNCOMPRESS;
      const uint32_t id = ((uint32_t)src[2] << 24) | ((uint32_t)src[3] << 16) | ((uint32_t)src[4] << 8) | src[5];
      if (id != *dict_id) return ZB_ERR_DICTIONARY;
      pos = 6;
    }
    expect = ((uint32_t)src[len - 4] << 24) | ((uint32_t)src[len - 3] << 16) | ((uint32_t)src[len - 2] << 8) | src[len - 1];
    return ZB_OK;
  }
  if (fmt == ZB_DF_DEFLATE) {
    if (raw_pos > len) return ZB_ERR_END_OF_BUFFER;
    pos = raw_pos;
    return ZB_OK;
  }
  return ZB_ERR_INVALID_FORMAT;
}

