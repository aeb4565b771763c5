// TEST SCAFFOLDING: the single-input deflate seam (zb200_deflate_bound, zb200_deflate) over the zlib-backed
// zb200_compress_batch of mock_abi_zlib.cpp, so that zippy::compress -- and the tarball writer of
// include/zippy_b200_tar.hpp -- can run on a machine without a GPU (tests/test_tarball_write.py).
// Linked together with mock_abi_zlib.cpp; never linked into the product.
#include <zlib.h>

#include "../../include/zippy_b200.h"

extern "C" {
size_t zb200_deflate_bound(size_t len) { return compressBound((uLong)len) + 64; }
int zb200_deflate(zb200_ctx *ctx, const uint8_t *src, size_t len, int level, uint8_t *dst, size_t dst_cap,
                  size_t *dst_len) {
  uint64_t so[2] = {0, len}, dof[2] = {0, 0};
  int st = 0;
  uint8_t dummy = 0;
  const int rc = zb200_compress_batch(ctx, src ? src : &dummy, so, 1, level, ZB200_DF_DEFLATE, nullptr, dst, dst_cap,
                                      dof, &st);
  if (rc) return rc;
  *dst_len = (size_t)dof[1];
  return st;
}
}
