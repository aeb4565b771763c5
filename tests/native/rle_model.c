/* rle_model.c -- a sequential CPU model of the run-length parse (ZB200_STRATEGY_RLE, k_lz<2>).
 *
 * An independent restatement of the rule in include/zippy_b200.h ("compression strategies"); it includes nothing
 * from the kernel.  It walks a member left to right, greedily, and writes the tokens in lz2_model.c's form:
 *   a literal byte b   -> b                  (< 256)
 *   a match            -> length << 16 | 1   (length 3..258, distance 1)
 * At position p, let e be the end of what p may reach: with cuts, the end of p's 4 KiB piece (pieces start at every
 * 64 KiB chunk start); without cuts, the member's end.  p starts a match when p has a byte before it (with cuts: p
 * is not its chunk's first byte) and M[p] = M[p + 1] = M[p + 2] = M[p - 1], all before e; its length is the longest
 * run of M[p - 1] from p, at most 258 and at most e - p.  Otherwise p is a literal.  Without cuts this is zlib
 * 1.3's deflate_rle. */
#include <stdint.h>

#ifdef __cplusplus
#define EXPORT extern "C"
#else
#define EXPORT
#endif

enum { CHUNK = 65536, PIECE = 4096, MAXM = 258 };

/* chunk_ntok[k] receives the number of tokens of chunk k (cuts only; room for max(1, ceil(n / 65536)) entries).
 * Returns the number of tokens, or -1 when `cap` is too small (nothing beyond cap is written). */
EXPORT int64_t rle_model(const uint8_t *m, uint64_t n, int cuts, uint32_t *tok, uint64_t cap, uint32_t *chunk_ntok) {
  uint64_t nt = 0, chunk_first = 0;
  uint32_t k = 0;
  if (cuts && chunk_ntok) chunk_ntok[0] = 0;
  for (uint64_t p = 0; p < n;) {
    const uint64_t c0 = cuts ? p / CHUNK * CHUNK : 0;
    if (cuts && c0 / CHUNK != k) {
      if (chunk_ntok) chunk_ntok[k] = (uint32_t)(nt - chunk_first);
      k = (uint32_t)(c0 / CHUNK);
      chunk_first = nt;
    }
    const uint64_t e = cuts ? (p / PIECE + 1) * PIECE < n ? (p / PIECE + 1) * PIECE : n : n;
    uint32_t t = m[p], len = 1;
    if (p > c0 && p + 3 <= e && m[p] == m[p - 1] && m[p + 1] == m[p - 1] && m[p + 2] == m[p - 1]) {
      const uint64_t lim = e - p < MAXM ? e - p : MAXM;
      len = 3;
      while (len < lim && m[p + len] == m[p - 1]) len++;
      t = len << 16 | 1u;
    }
    if (nt < cap) tok[nt] = t;
    nt++;
    p += len;
  }
  if (cuts && chunk_ntok) chunk_ntok[k] = (uint32_t)(nt - chunk_first);
  return nt > cap ? -1 : (int64_t)nt;
}
