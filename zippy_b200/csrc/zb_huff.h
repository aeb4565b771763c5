// zb_huff.h -- per-chunk Huffman code construction (host + device).
//
// Replaces the reference's huffmanCodes (src/zippy/deflate.nim:13-151, heap of GC'd
// nodes + heuristic rebalancing) and its dynamic-header writer (deflate.nim:295-394)
// with a single-thread, allocation-free formulation: sort used symbols, Moffat-
// Katajainen in-place minimum-redundancy lengths, Kraft-sum length limiting, canonical
// LSB-first codes, code-length RLE, and exact bit accounting so the packer never needs
// a sizing pass.  This is the host builder and the reference: k_huff (zb_huff_warp.cuh) builds
// the same codebook with one warp per chunk in parallel stages (1.37 ms for C2's 65 536 chunks
// on an H100 80GB HBM3 at 700 W, against 3.41 ms for this code on one GPU thread per chunk), and
// tests/test_gpu_huff_identity.py compares the two byte for byte; tests/test_host_units.py pins
// this code's codebooks.
#pragma once
#include "zb_common.h"

struct ZbCodebook {
  uint32_t ll[288];          // litlen: code (bit-reversed, emit LSB-first) | len << 16
  uint32_t dd[32];           // distance: same packing
  uint32_t block_type;       // 0 stored, 1 fixed, 2 dynamic
  uint32_t hdr_bits;         // bits in hdr[] (block header + dynamic tables)
  uint32_t warp_bit_start[ZB_WARPS_PER_CHUNK];  // bit offset inside the chunk's output
  uint32_t eob_bit_start;    // where the end-of-block code goes
  uint32_t total_bytes;      // bytes this chunk occupies in the member's deflate stream
  uint32_t is_final;         // BFINAL set on this chunk's (last) block
  uint32_t chunk_len;        // input bytes
  uint8_t hdr[336];          // header bits, LSB-first
};

// Fixed-Huffman code lengths (RFC 1951 3.2.6; reference internal.nim:151-175).
ZB_HD int zb_fixed_ll_len(int s) { return s <= 143 ? 8 : s <= 255 ? 9 : s <= 279 ? 7 : 8; }

// Canonical codes from lengths (RFC 1951 3.2.2), bit-reversed for LSB-first emission
// (reference deflate.nim:136-149 / internal.nim:133-149).  out[i] = code | len<<16.
ZB_HD_NOINLINE void zb_canonical_codes(const uint8_t *lens, int n, uint32_t *out) {
  uint32_t count[16];
  uint32_t next[16];
  for (int i = 0; i < 16; i++) count[i] = 0;
  for (int i = 0; i < n; i++) count[lens[i]]++;
  count[0] = 0;
  next[0] = 0;
  for (int l = 1; l < 16; l++) next[l] = (next[l - 1] + count[l - 1]) << 1;
  for (int i = 0; i < n; i++) {
    int l = lens[i];
    out[i] = l ? (zb_brev16(next[l]++, l) | ((uint32_t)l << 16)) : 0u;
  }
}

// Length-limited Huffman code lengths for freq[0..n); always a COMPLETE code
// (zlib rejects incomplete literal/length sets).  0 or 1 used symbols follow the
// reference's convention (deflate.nim:34-45): two codes of length 1.
ZB_HD_NOINLINE void zb_huff_lengths(const uint32_t *freq, int n, int limit, uint8_t *lens) {
  uint32_t key[ZB_NUM_LITLEN];  // freq << 9 | symbol, sorted ascending
  uint32_t a[ZB_NUM_LITLEN];
  int m = 0;
  for (int i = 0; i < n; i++) {
    lens[i] = 0;
    if (freq[i]) key[m++] = (freq[i] << 9) | (uint32_t)i;
  }
  if (m == 0) {
    lens[0] = 1;
    lens[1] = 1;
    return;
  }
  if (m == 1) {
    int s = (int)(key[0] & 511u);
    lens[s] = 1;
    lens[s == 0 ? 1 : 0] = 1;
    return;
  }
  // ascending by (frequency, symbol): the keys are in symbol order already, so a STABLE sort on the frequency
  // alone does it -- 6-bit counting passes through `a` (frequencies are below 2^17: a chunk is 64 KiB; the
  // code-length alphabet's below 2^9).  (A shell sort was a third of this routine's instructions.)
  {
    uint32_t maxf = 0;
    for (int i = 0; i < m; i++) maxf |= key[i] >> 9;
    uint32_t *from = key, *to = a;
    for (int shift = 9; (maxf >> (shift - 9)) != 0u; shift += 6) {
      uint16_t cnt6[64];
      for (int b = 0; b < 64; b++) cnt6[b] = 0;
      for (int i = 0; i < m; i++) cnt6[(from[i] >> shift) & 63u]++;
      uint16_t run = 0;
      for (int b = 0; b < 64; b++) {
        const uint16_t c = cnt6[b];
        cnt6[b] = run;
        run = (uint16_t)(run + c);
      }
      for (int i = 0; i < m; i++) to[cnt6[(from[i] >> shift) & 63u]++] = from[i];
      uint32_t *t = from;
      from = to;
      to = t;
    }
    if (from != key)
      for (int i = 0; i < m; i++) key[i] = from[i];
  }
  for (int i = 0; i < m; i++) a[i] = key[i] >> 9;
  // Moffat & Katajainen, "In-place calculation of minimum-redundancy codes" (1995)
  if (m == 2) {
    a[0] = a[1] = 1;
  } else {
    a[0] += a[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < m - 1; next++) {
      if (leaf >= m || a[root] < a[leaf]) {
        a[next] = a[root];
        a[root++] = (uint32_t)next;
      } else {
        a[next] = a[leaf++];
      }
      if (leaf >= m || (root < next && a[root] < a[leaf])) {
        a[next] += a[root];
        a[root++] = (uint32_t)next;
      } else {
        a[next] += a[leaf++];
      }
    }
    a[m - 2] = 0;
    for (int next = m - 3; next >= 0; next--) a[next] = a[a[next]] + 1;
    int avbl = 1, used = 0, dpth = 0, root2 = m - 2, next = m - 1;
    while (avbl > 0) {
      while (root2 >= 0 && (int)a[root2] == dpth) {
        used++;
        root2--;
      }
      while (avbl > used) {
        a[next--] = (uint32_t)dpth;
        avbl--;
      }
      avbl = 2 * used;
      dpth++;
      used = 0;
    }
  }
  // a[i] = optimal depth of the i-th least frequent symbol (non-increasing in i).
  // Length limiting on the per-length counts: clamp, then repair the Kraft sum one
  // unit at a time (each step keeps the symbol count and lowers the sum by 2^-limit).
  uint32_t num[33];
  for (int i = 0; i <= 32; i++) num[i] = 0;
  for (int i = 0; i < m; i++) num[a[i] > 32 ? 32 : a[i]]++;
  for (int l = limit + 1; l <= 32; l++) {
    num[limit] += num[l];
    num[l] = 0;
  }
  uint32_t total = 0;
  for (int l = limit; l >= 1; l--) total += num[l] << (limit - l);
  while (total > (1u << limit)) {
    num[limit]--;
    for (int l = limit - 1; l >= 1; l--)
      if (num[l]) {
        num[l]--;
        num[l + 1] += 2;
        break;
      }
    total--;
  }
  int idx = 0;  // least frequent first -> longest codes first
  for (int l = limit; l >= 1; l--)
    for (uint32_t c = 0; c < num[l]; c++) lens[key[idx++] & 511u] = (uint8_t)l;
}

struct ZbBitSink {
  uint8_t *p;
  uint32_t nbits;
};
ZB_HD void zb_put_bits(ZbBitSink *s, uint32_t v, int n) {  // n <= 16, LSB first; whole bytes at a time
  uint32_t pos = s->nbits;
  s->nbits += (uint32_t)n;
  v &= (1u << n) - 1u;
  while (n > 0) {
    const uint32_t sh = pos & 7u, take = 8u - sh < (uint32_t)n ? 8u - sh : (uint32_t)n;
    const uint8_t old = sh ? s->p[pos >> 3] : (uint8_t)0;
    s->p[pos >> 3] = (uint8_t)(old | ((v & ((1u << take) - 1u)) << sh));
    v >>= take;
    pos += take;
    n -= (int)take;
  }
}

// Build everything the packer needs for one chunk.
//   hist: per-warp histograms, hist[w * ZB_HIST_SYMS + s], s < 286 literal/length,
//         s >= 286 distance codes; end-of-block is NOT counted (added here).
//   force_type: -1 choose smallest, 0 force stored (level 0), 1 the smaller of stored and fixed, never dynamic
//   (ZB200_STRATEGY_FIXED).
ZB_HD_NOINLINE void zb_build_codebook(const uint16_t *hist, uint32_t chunk_len, int is_final,
                                      int force_type, ZbCodebook *cb) {
  const uint8_t len_extra[29] = ZB_LENGTH_EXTRA;
  const uint8_t dist_extra[30] = ZB_DIST_EXTRA;
  const uint8_t clcl_order[19] = ZB_CLCL_ORDER;
  // (the histograms are pairs of 16-bit counters in 32-bit words -- ZB_HIST_SYMS is even and every sub-chunk's
  // histogram starts on a word -- so they are read a word at a time)
  uint32_t llf[ZB_NUM_LITLEN], df[ZB_NUM_DIST];
  const uint32_t *hw = reinterpret_cast<const uint32_t *>(hist);
  for (int p2 = 0; p2 < ZB_HIST_SYMS / 2; p2++) {
    uint32_t lo = 0, hi = 0;
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
      const uint32_t v = hw[w * (ZB_HIST_SYMS / 2) + p2];
      lo += v & 0xffffu;
      hi += v >> 16;
    }
    const int s0 = 2 * p2;
    if (s0 < ZB_NUM_LITLEN) llf[s0] = lo; else df[s0 - ZB_NUM_LITLEN] = lo;
    if (s0 + 1 < ZB_NUM_LITLEN) llf[s0 + 1] = hi; else df[s0 + 1 - ZB_NUM_LITLEN] = hi;
  }
  llf[256] = 1;
  cb->is_final = (uint32_t)is_final;
  cb->chunk_len = chunk_len;

  // --- dynamic code ---
  uint8_t lens[ZB_NUM_LITLEN + ZB_NUM_DIST];
  zb_huff_lengths(llf, ZB_NUM_LITLEN, 15, lens);
  zb_huff_lengths(df, ZB_NUM_DIST, 15, lens + ZB_NUM_LITLEN);
  int nll = ZB_NUM_LITLEN, nd = ZB_NUM_DIST;
  while (nll > 257 && lens[nll - 1] == 0) nll--;
  while (nd > 1 && lens[ZB_NUM_LITLEN + nd - 1] == 0) nd--;
  // (32-bit sums: at most 65 537 tokens of at most 48 bits)
  uint32_t dyn_payload32 = 0, fix_payload32 = 0, extra32 = 0;
  for (int s = 0; s < ZB_NUM_LITLEN; s++) {
    dyn_payload32 += llf[s] * lens[s];
    fix_payload32 += llf[s] * (uint32_t)zb_fixed_ll_len(s);
    if (s > 256) extra32 += llf[s] * len_extra[s - 257];
  }
  for (int s = 0; s < ZB_NUM_DIST; s++) {
    dyn_payload32 += df[s] * lens[ZB_NUM_LITLEN + s];
    fix_payload32 += df[s] * 5u;
    extra32 += df[s] * dist_extra[s];
  }
  const uint64_t dyn_payload = dyn_payload32, fix_payload = fix_payload32, extra = extra32;
  // code-length sequence -> RLE symbols (RFC 1951 3.2.7)
  uint8_t seq[ZB_NUM_LITLEN + ZB_NUM_DIST];
  int nseq = 0;
  for (int i = 0; i < nll; i++) seq[nseq++] = lens[i];
  for (int i = 0; i < nd; i++) seq[nseq++] = lens[ZB_NUM_LITLEN + i];
  uint8_t rsym[ZB_NUM_LITLEN + ZB_NUM_DIST], rext[ZB_NUM_LITLEN + ZB_NUM_DIST];
  int nr = 0;
  uint32_t clf[19];
  for (int i = 0; i < 19; i++) clf[i] = 0;
  for (int i = 0; i < nseq;) {
    int v = seq[i], run = 1;
    while (i + run < nseq && seq[i + run] == v) run++;
    int left = run;
    if (v == 0) {
      while (left >= 11) {
        int r = left > 138 ? 138 : left;
        rsym[nr] = 18;
        rext[nr++] = (uint8_t)(r - 11);
        left -= r;
      }
      if (left >= 3) {
        rsym[nr] = 17;
        rext[nr++] = (uint8_t)(left - 3);
        left = 0;
      }
      while (left-- > 0) {
        rsym[nr] = 0;
        rext[nr++] = 0;
      }
    } else {
      rsym[nr] = (uint8_t)v;
      rext[nr++] = 0;
      left--;
      while (left >= 3) {
        int r = left > 6 ? 6 : left;
        rsym[nr] = 16;
        rext[nr++] = (uint8_t)(r - 3);
        left -= r;
      }
      while (left-- > 0) {
        rsym[nr] = (uint8_t)v;
        rext[nr++] = 0;
      }
    }
    i += run;
  }
  for (int i = 0; i < nr; i++) clf[rsym[i]]++;
  uint8_t cll[19];
  zb_huff_lengths(clf, 19, 7, cll);
  uint32_t clc[19];
  zb_canonical_codes(cll, 19, clc);
  int hclen = 19;
  while (hclen > 4 && cll[clcl_order[hclen - 1]] == 0) hclen--;
  uint32_t dyn_hdr = 3 + 5 + 5 + 4 + 3u * (uint32_t)hclen;
  for (int i = 0; i < nr; i++)
    dyn_hdr += cll[rsym[i]] + (rsym[i] == 16 ? 2u : rsym[i] == 17 ? 3u : rsym[i] == 18 ? 7u : 0u);

  uint64_t dyn_bits = dyn_hdr + dyn_payload + extra;
  uint64_t fix_bits = 3 + fix_payload + extra;
  uint32_t npieces = chunk_len == 0 ? 1u : (chunk_len + 65534u) / 65535u;
  uint64_t stored_bytes = (uint64_t)chunk_len + 5ull * npieces;
  // bytes for a coded block: payload, then either pad-to-byte (final) or an empty
  // stored block as a byte-aligning sync marker (3 bits + pad + 00 00 ff ff).
  uint64_t dyn_bytes = is_final ? (dyn_bits + 7) / 8 : (dyn_bits + 3 + 7) / 8 + 4;
  uint64_t fix_bytes = is_final ? (fix_bits + 7) / 8 : (fix_bits + 3 + 7) / 8 + 4;

  int type = 2;
  uint64_t best = dyn_bytes;
  if (fix_bytes < best || force_type == 1) {
    type = 1;
    best = fix_bytes;
  }
  if (stored_bytes <= best) {
    type = 0;
    best = stored_bytes;
  }
  if (force_type == 0) {
    type = 0;
    best = stored_bytes;
  }
  cb->block_type = (uint32_t)type;
  cb->total_bytes = (uint32_t)best;

  ZbBitSink sink;
  sink.p = cb->hdr;
  sink.nbits = 0;
  if (type == 0) {
    cb->hdr_bits = 0;
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) cb->warp_bit_start[w] = 0;
    cb->eob_bit_start = 0;
    return;
  }
  uint8_t use_lens[ZB_NUM_LITLEN + 2 + ZB_NUM_DIST + 2];
  if (type == 1) {
    zb_put_bits(&sink, (uint32_t)(is_final ? 1 : 0), 1);
    zb_put_bits(&sink, 1, 2);
    for (int s = 0; s < 288; s++) use_lens[s] = (uint8_t)zb_fixed_ll_len(s);
    zb_canonical_codes(use_lens, 288, cb->ll);
    for (int s = 0; s < 32; s++) use_lens[s] = 5;
    zb_canonical_codes(use_lens, 32, cb->dd);
    for (int s = 0; s < ZB_NUM_LITLEN; s++) lens[s] = (uint8_t)zb_fixed_ll_len(s);
    for (int s = 0; s < ZB_NUM_DIST; s++) lens[ZB_NUM_LITLEN + s] = 5;
  } else {
    zb_put_bits(&sink, (uint32_t)(is_final ? 1 : 0), 1);
    zb_put_bits(&sink, 2, 2);
    zb_put_bits(&sink, (uint32_t)(nll - 257), 5);
    zb_put_bits(&sink, (uint32_t)(nd - 1), 5);
    zb_put_bits(&sink, (uint32_t)(hclen - 4), 4);
    for (int i = 0; i < hclen; i++) zb_put_bits(&sink, cll[clcl_order[i]], 3);
    for (int i = 0; i < nr; i++) {
      zb_put_bits(&sink, clc[rsym[i]] & 0xffffu, (int)(clc[rsym[i]] >> 16));
      if (rsym[i] == 16) zb_put_bits(&sink, rext[i], 2);
      else if (rsym[i] == 17) zb_put_bits(&sink, rext[i], 3);
      else if (rsym[i] == 18) zb_put_bits(&sink, rext[i], 7);
    }
    zb_canonical_codes(lens, ZB_NUM_LITLEN, cb->ll);
    cb->ll[286] = cb->ll[287] = 0;
    zb_canonical_codes(lens + ZB_NUM_LITLEN, ZB_NUM_DIST, cb->dd);
    cb->dd[30] = cb->dd[31] = 0;
  }
  cb->hdr_bits = sink.nbits;
  // per-warp token bit ranges
  // (one cost per symbol = code length + extra bits, in histogram order, so the eight sums are plain dot products)
  uint8_t cost[ZB_HIST_SYMS];
  for (int s = 0; s < ZB_NUM_LITLEN; s++) cost[s] = (uint8_t)(lens[s] + (s > 256 ? len_extra[s - 257] : 0));
  for (int s = 0; s < ZB_NUM_DIST; s++) cost[ZB_NUM_LITLEN + s] = (uint8_t)(lens[ZB_NUM_LITLEN + s] + dist_extra[s]);
  uint32_t pos = sink.nbits;
  for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
    cb->warp_bit_start[w] = pos;
    const uint32_t *h2 = hw + w * (ZB_HIST_SYMS / 2);
    uint32_t bits = 0;
    for (int p2 = 0; p2 < ZB_HIST_SYMS / 2; p2++) {
      const uint32_t v = h2[p2];
      bits += (v & 0xffffu) * cost[2 * p2] + (v >> 16) * cost[2 * p2 + 1];
    }
    pos += bits;
  }
  cb->eob_bit_start = pos;
}
