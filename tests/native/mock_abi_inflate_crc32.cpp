// TEST SCAFFOLDING: zb200_inflate_batch_crc32 over zlib, so that the ZipArchive reader of
// include/zippy_b200_zip.hpp can run on a machine without a GPU (tests/test_ziparchive_v1.py).  Linked together
// with mock_abi_zlib.cpp; never linked into the product.
#include <zlib.h>

#include <cstring>

#include "../../include/zippy_b200.h"

extern "C" {
int zb200_inflate_batch_crc32(zb200_ctx *, const uint8_t *base, const uint64_t *off, size_t n, uint8_t *dst,
                              const uint64_t *dst_off, uint64_t *lens, uint32_t *crcs, int *st) {
  for (size_t i = 0; i < n; i++) {
    z_stream zs;
    std::memset(&zs, 0, sizeof(zs));
    if (inflateInit2(&zs, -15) != Z_OK) return ZB200_ERR_UNCOMPRESS;
    zs.next_in = const_cast<Bytef *>(base + off[i]);
    zs.avail_in = (uInt)(off[i + 1] - off[i]);
    zs.next_out = dst + dst_off[i];
    zs.avail_out = (uInt)(dst_off[i + 1] - dst_off[i]);
    const int rc = inflate(&zs, Z_FINISH);
    const bool ok = rc == Z_STREAM_END;
    st[i] = ok ? ZB200_OK : (rc == Z_BUF_ERROR && zs.avail_out == 0) ? ZB200_ERR_DST_TOO_SMALL : ZB200_ERR_UNCOMPRESS;
    lens[i] = ok ? zs.total_out : 0;
    crcs[i] = ok ? (uint32_t)crc32(0L, dst + dst_off[i], (uInt)zs.total_out) : 0;
    inflateEnd(&zs);
  }
  return ZB200_OK;
}
}
