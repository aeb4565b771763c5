// zb_huff_warp.cuh -- k_huff: one warp per chunk builds the chunk's ZbCodebook (zb_huff.h) in shared memory.
//
// The result is bit for bit what the host builder zb_build_codebook writes into a zero-filled ZbCodebook (the
// tests compare the two): every word of the struct is stored, and the fields the host builder leaves alone are
// 0 here -- ll[], dd[] and hdr[] of a stored block, and hdr[] past the byte that holds the header's last bit.
// The keys freq << 9 | symbol are distinct, so any exact sort gives the serial counting sort's order; every step
// but the Moffat-Katajainen walk is a data-parallel function of that order and the counts.  Stages:
//   sum     the eight sub-chunk histograms, coalesced word loads, two symbol counts per word in registers
//   sort    used symbols compacted by ballot; ranked by counting (literal/length keys before distance keys)
//   mk      Moffat-Katajainen in shared memory: lane 0 the literal/length alphabet, lane 1 the distance alphabet,
//           the same instructions at the same time; the leaf depths are counted per depth, not stored
//   limit   Kraft repair of the per-length counts, on the same two lanes
//   assign  code lengths from the prefix of the per-length counts; payload and extra-bit sums as warp reductions
//   rle     the code-length sequence as RLE symbols, serial on lane 0 (at most 316 entries)
//   cl      the 19-symbol code-length code: sort, Moffat-Katajainen and limit on lane 0, canonical codes
//   header  block choice; header fields placed by a prefix sum of their widths, OR-ed into a staging copy
//   codes   canonical codes: per-length counts and ranks among equal lengths by __match_any_sync and popc
//   bits    the eight sub-chunk bit ranges: dot products of the histograms with the per-symbol cost (the histogram
//           words are read again; they were read a few microseconds before and come from L2)
//   store   scalars and header: coalesced word stores
// -DZB_HUFF_STAGE_CLOCKS=1 (a diagnostic build, never the shipped one; tools/lz1_stages.py --kernel huff makes it):
// lane 0 of every warp adds the clock64() cycles of each stage into zb_huff_stage_clk, read back (and zeroed) by
// zb200_huff_stage_clocks.  The stage order is the one HUFF_STAGE_NAMES in that tool prints.
#pragma once
#include <stddef.h>

#include "zb_device.cuh"
#include "zb_kernels.h"

#define HW_WARPS 4  // chunks (warps) per CTA

static_assert(offsetof(ZbCodebook, dd) == 288 * 4 && offsetof(ZbCodebook, block_type) == 320 * 4 &&
                  offsetof(ZbCodebook, warp_bit_start) == 322 * 4 && offsetof(ZbCodebook, chunk_len) == 333 * 4 &&
                  offsetof(ZbCodebook, hdr) == 334 * 4 && sizeof(ZbCodebook) == 418 * 4,
              "k_huff stores the codebook as 418 words: ll, dd, 14 scalars, 84 header words");
#define HW_TAIL_WORDS (418 - 320)  // block_type .. hdr

// Per-warp workspace.  `key` holds the sort input, then (from the RLE on) the RLE symbols and the code-length
// code's arrays (HW_K_*); `skey` holds the sorted keys, then (from the header on) the staging copy of the
// codebook's tail and the canonical-code tables (HW_S_*).
struct __align__(16) HwWarp {
  uint32_t key[320];   // used symbols' keys (distance keys with bit 31 set), padded with 0xffffffff
  uint32_t skey[320];  // ascending
  uint32_t a[320];     // Moffat-Katajainen's array
  uint8_t lens[320];   // literal/length code lengths [0, 288), distance [288, 320)
  uint32_t num_ll[36], num_d[36];  // per-length counts (index = length)
  uint32_t clf[20];    // code-length symbol frequencies
};
#define HW_K_RSYM 0      // bytes [0, 316)
#define HW_K_REXT 80     // bytes [320, 636)
#define HW_K_CKEY 160    // [24]
#define HW_K_CSKEY 184   // [24]
#define HW_K_CA 208      // [24]
#define HW_K_NUMC 232    // [36]
#define HW_K_CLL 268     // 20 bytes
#define HW_K_CLC 276     // [20]
static_assert(HW_K_CLC + 20 <= 320, "code-length arrays fit in key[]");
#define HW_S_TAIL 0      // [98]
#define HW_S_CNT 100     // [16]
#define HW_S_NXT 116     // [16]

#ifndef ZB_HUFF_STAGE_CLOCKS
#define ZB_HUFF_STAGE_CLOCKS 0
#endif
enum { HWS_SUM, HWS_SORT, HWS_MK, HWS_LIMIT, HWS_ASSIGN, HWS_RLE, HWS_CL, HWS_HEADER, HWS_CODES, HWS_BITS, HWS_STORE, HWS_N };
#if ZB_HUFF_STAGE_CLOCKS
__device__ unsigned long long zb_huff_stage_clk[HWS_N];
#endif
struct HwClk {
#if ZB_HUFF_STAGE_CLOCKS
  unsigned long long acc[HWS_N];
  long long t;
  __device__ __forceinline__ void start() {
#pragma unroll
    for (int s = 0; s < HWS_N; s++) acc[s] = 0;
    t = clock64();
  }
  __device__ __forceinline__ void mark(int s) {
    const long long n = clock64();
    acc[s] += (unsigned long long)(n - t);
    t = n;
  }
  __device__ __forceinline__ void publish() {
    if (zb_lane() == 0)
#pragma unroll
      for (int s = 0; s < HWS_N; s++) atomicAdd(&zb_huff_stage_clk[s], acc[s]);
  }
#else
  __device__ __forceinline__ void start() {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void publish() {}
#endif
};

// Moffat & Katajainen (as zb_huff_lengths) on a[0..m) = ascending frequencies, one lane: num[d] = the number of
// leaves at depth d (depths past 32 counted at 32), num[] zeroed first.  m < 2 leaves num[] zero.
__device__ __forceinline__ void hw_mk(uint32_t *a, int m, uint32_t *num) {
  for (int i = 0; i <= 32; i++) num[i] = 0;
  if (m < 2) return;
  if (m == 2) {
    num[1] = 2;
    return;
  }
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
  // a[0..m-2] = depths of the internal nodes, non-increasing; at each depth the nodes not internal are leaves
  int avbl = 1, used = 0, dpth = 0, root2 = m - 2;
  while (avbl > 0) {
    while (root2 >= 0 && (int)a[root2] == dpth) {
      used++;
      root2--;
    }
    if (avbl > used) num[dpth > 32 ? 32 : dpth] += (uint32_t)(avbl - used);
    avbl = 2 * used;
    dpth++;
    used = 0;
  }
}

// zb_huff_lengths' length limiting on the per-length counts, one lane
__device__ __forceinline__ void hw_limit(uint32_t *num, int m, int limit) {
  if (m < 2) return;
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
}

// the code length of the j-th least frequent of m >= 2 symbols: longest codes first
__device__ __forceinline__ uint32_t hw_len_at(const uint32_t *num, int limit, uint32_t j) {
  uint32_t l = (uint32_t)limit, c = num[limit];
  while (j >= c) c += num[--l];
  return l;
}

// OR the n <= 16 bits v at bit `bit` of the LSB-first word array w
__device__ __forceinline__ void hw_or_bits(uint32_t *w, uint32_t bit, uint32_t v, uint32_t n) {
  const uint32_t sh = bit & 31u;
  atomicOr(&w[bit >> 5], v << sh);
  if (sh + n > 32u) atomicOr(&w[(bit >> 5) + 1], v >> (32u - sh));
}

// zb_canonical_codes of lens[0..n), whole warp; cnt, nxt: 16 words of scratch each
__device__ __forceinline__ void hw_canon(const uint8_t *lens, int n, uint32_t *out, uint32_t *cnt, uint32_t *nxt) {
  const int lane = zb_lane();
  const uint32_t lt = (1u << lane) - 1u;
  if (lane < 16) cnt[lane] = 0;
  __syncwarp();
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const uint32_t l = s < n ? lens[s] : 0u;
    const uint32_t peers = __match_any_sync(ZB_FULL, l);
    if (l && lane == 31 - __clz((int)peers)) cnt[l] += (uint32_t)__popc(peers);
    __syncwarp();
  }
  if (lane >= 1 && lane < 16) {
    uint32_t nx = 0;
    for (int k = 1; k < lane; k++) nx = (nx + cnt[k]) << 1;
    nxt[lane] = nx;
  }
  __syncwarp();
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const uint32_t l = s < n ? lens[s] : 0u;
    const uint32_t peers = __match_any_sync(ZB_FULL, l);
    const uint32_t code = l ? nxt[l] + (uint32_t)__popc(peers & lt) : 0u;
    __syncwarp();
    if (l && lane == 31 - __clz((int)peers)) nxt[l] += (uint32_t)__popc(peers);
    __syncwarp();
    if (s < n) out[s] = l ? (zb_brev16(code, (int)l) | (l << 16)) : 0u;
  }
}

// the bits a token of histogram symbol s costs: code length + extra bits
__device__ __forceinline__ uint32_t hw_cost(const uint8_t *lens, int s) {
  return s < ZB_NUM_LITLEN ? lens[s] + (s > 256 ? (uint32_t)zb_len_extra_bits(s - 257) : 0u)
                           : lens[288 + s - ZB_NUM_LITLEN] + (uint32_t)zb_dist_extra_bits(s - ZB_NUM_LITLEN);
}

//   hw: the chunk's eight sub-chunk histograms as words (two u16 counters each), end-of-block not counted
//   force_type: -1 choose the smallest block, 0 stored (level 0), 1 the smaller of stored and fixed (never dynamic)
__device__ __forceinline__ void hw_build_codebook(HwWarp &ws, const uint32_t *__restrict__ hw, uint32_t chunk_len,
                                                  uint32_t is_final, int force_type, ZbCodebook *cb, HwClk &clk) {
  const int lane = zb_lane();
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t *gw = reinterpret_cast<uint32_t *>(cb);
  const uint32_t npieces = chunk_len == 0 ? 1u : (chunk_len + 65534u) / 65535u;
  const uint64_t stored_bytes = (uint64_t)chunk_len + 5ull * npieces;
  if (force_type == 0) {
    for (int i = lane; i < 418; i += 32)
      gw[i] = i == 331 ? (uint32_t)stored_bytes : i == 332 ? is_final : i == 333 ? chunk_len : 0u;
    return;
  }

  // ---- sum ----
  uint32_t fa[5], fb[5];  // counts of symbols 2p, 2p + 1 for p = lane + 32k
#pragma unroll
  for (int k = 0; k < 5; k++) {
    const int p = lane + 32 * k;
    uint32_t lo = 0, hi = 0;
    if (p < ZB_HIST_WORDS)
#pragma unroll
      for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
        const uint32_t v = __ldg(hw + w * ZB_HIST_WORDS + p);
        lo += v & 0xffffu;
        hi += v >> 16;
      }
    fa[k] = p == 128 ? 1u : lo;  // end-of-block, symbol 256: once (as the host builder, whatever the histogram holds)
    fb[k] = hi;
  }
  {
    uint32_t *l32 = reinterpret_cast<uint32_t *>(ws.lens);
    for (int i = lane; i < 80; i += 32) l32[i] = 0;
  }
  clk.mark(HWS_SUM);

  // ---- sort ----
  int m = 0, mll = 0;
#pragma unroll
  for (int k = 0; k < 5; k++) {
    const uint32_t s0 = 2u * (uint32_t)(lane + 32 * k);
    const bool u0 = fa[k] != 0, u1 = fb[k] != 0;
    const uint32_t b0 = __ballot_sync(ZB_FULL, u0), b1 = __ballot_sync(ZB_FULL, u1);
    const int at = m + __popc(b0 & lt) + __popc(b1 & lt);
    const bool isd = s0 >= ZB_NUM_LITLEN;
    const uint32_t kb = (isd ? 0x80000000u : 0u) | (isd ? s0 - ZB_NUM_LITLEN : s0);
    if (u0) ws.key[at] = kb | (fa[k] << 9);
    if (u1) ws.key[at + (u0 ? 1 : 0)] = (kb + 1u) | (fb[k] << 9);
    m += __popc(b0) + __popc(b1);
    const uint32_t llm = k < 4 ? ZB_FULL : 0x7fffu;  // words below 143 hold literal/length symbols
    mll += __popc(b0 & llm) + __popc(b1 & llm);
  }
  if (lane < 4) ws.key[m + lane] = 0xffffffffu;
  __syncwarp();
  {
    const uint4 *q4 = reinterpret_cast<const uint4 *>(ws.key);
    const int nq = (m + 3) >> 2;
    for (int base = 0; base < m; base += 64) {
      const int i0 = base + lane, i1 = i0 + 32;
      const uint32_t k0 = i0 < m ? ws.key[i0] : 0u, k1 = i1 < m ? ws.key[i1] : 0u;
      uint32_t r0 = 0, r1 = 0;
      for (int j = 0; j < nq; j++) {
        const uint4 q = q4[j];
        r0 += (uint32_t)(q.x < k0) + (uint32_t)(q.y < k0) + (uint32_t)(q.z < k0) + (uint32_t)(q.w < k0);
        r1 += (uint32_t)(q.x < k1) + (uint32_t)(q.y < k1) + (uint32_t)(q.z < k1) + (uint32_t)(q.w < k1);
      }
      if (i0 < m) ws.skey[r0] = k0;
      if (i1 < m) ws.skey[r1] = k1;
    }
  }
  __syncwarp();
  for (int i = lane; i < m; i += 32) ws.a[i] = (ws.skey[i] >> 9) & 0x3fffffu;
  __syncwarp();
  clk.mark(HWS_SORT);

  // ---- Moffat-Katajainen and limit: literal/length on lane 0, distance on lane 1 ----
  const int md = m - mll;
  if (lane < 2) hw_mk(lane ? ws.a + mll : ws.a, lane ? md : mll, lane ? ws.num_d : ws.num_ll);
  __syncwarp();
  clk.mark(HWS_MK);
  if (lane < 2) hw_limit(lane ? ws.num_d : ws.num_ll, lane ? md : mll, 15);
  __syncwarp();
  clk.mark(HWS_LIMIT);

  // ---- assign lengths; payload sums ----
  uint32_t dyn_payload, fix_payload, extra;
  {
    uint32_t dyn = 0, fix = 0, ext = 0;
    for (int i = lane; i < m; i += 32) {
      const uint32_t k = ws.skey[i];
      const bool isd = i >= mll;
      const int mx = isd ? md : mll;
      const uint32_t l = mx >= 2 ? hw_len_at(isd ? ws.num_d : ws.num_ll, 15, (uint32_t)(isd ? i - mll : i)) : 1u;
      const uint32_t f = (k >> 9) & 0x3fffffu, s = k & 511u;
      ws.lens[isd ? 288 + s : s] = (uint8_t)l;
      dyn += f * l;
      fix += f * (isd ? 5u : (uint32_t)zb_fixed_ll_len((int)s));
      ext += f * (uint32_t)(isd ? zb_dist_extra_bits((int)s) : s > 256 ? zb_len_extra_bits((int)s - 257) : 0);
    }
    if (lane == 0) {  // 0 or 1 used symbols: two codes of length 1
      if (mll < 2) {
        const uint32_t s = mll ? ws.skey[0] & 511u : 0u;
        ws.lens[s == 0 ? 1 : 0] = 1;
        if (!mll) ws.lens[0] = 1;
      }
      if (md < 2) {
        const uint32_t s = md ? ws.skey[mll] & 511u : 0u;
        ws.lens[288 + (s == 0 ? 1 : 0)] = 1;
        if (!md) ws.lens[288] = 1;
      }
    }
    dyn_payload = __reduce_add_sync(ZB_FULL, dyn);
    fix_payload = __reduce_add_sync(ZB_FULL, fix);
    extra = __reduce_add_sync(ZB_FULL, ext);
  }
  if (lane < 19) ws.clf[lane] = 0;
  __syncwarp();
  int nll, nd;
  {
    uint32_t hi = 0;
    for (int s = lane; s < ZB_NUM_LITLEN; s += 32)
      if (ws.lens[s]) hi = (uint32_t)s + 1u;
    nll = max(257, (int)__reduce_max_sync(ZB_FULL, hi));
    nd = max(1, (int)__reduce_max_sync(ZB_FULL, (lane < ZB_NUM_DIST && ws.lens[288 + lane]) ? (uint32_t)lane + 1u : 0u));
  }
  clk.mark(HWS_ASSIGN);

  // ---- RLE of the code-length sequence (RFC 1951 3.2.7), lane 0 ----
  uint8_t *rsym = reinterpret_cast<uint8_t *>(ws.key + HW_K_RSYM);
  uint8_t *rext = reinterpret_cast<uint8_t *>(ws.key + HW_K_REXT);
  int nr = 0;
  if (lane == 0) {
    const int nseq = nll + nd;
    auto seq = [&](int i) { return (int)ws.lens[i < nll ? i : 288 + i - nll]; };
    auto emit = [&](int sy, int ex) {
      rsym[nr] = (uint8_t)sy;
      rext[nr++] = (uint8_t)ex;
      ws.clf[sy]++;
    };
    for (int i = 0; i < nseq;) {
      const int v = seq(i);
      int run = 1;
      while (i + run < nseq && seq(i + run) == v) run++;
      int left = run;
      if (v == 0) {
        while (left >= 11) {
          const int r = left > 138 ? 138 : left;
          emit(18, r - 11);
          left -= r;
        }
        if (left >= 3) {
          emit(17, left - 3);
          left = 0;
        }
        while (left-- > 0) emit(0, 0);
      } else {
        emit(v, 0);
        left--;
        while (left >= 3) {
          const int r = left > 6 ? 6 : left;
          emit(16, r - 3);
          left -= r;
        }
        while (left-- > 0) emit(v, 0);
      }
      i += run;
    }
  }
  nr = __shfl_sync(ZB_FULL, nr, 0);
  __syncwarp();
  clk.mark(HWS_RLE);

  // ---- the code-length code ----
  uint32_t *ckey = ws.key + HW_K_CKEY, *cskey = ws.key + HW_K_CSKEY, *ca = ws.key + HW_K_CA, *num_c = ws.key + HW_K_NUMC;
  uint8_t *cll = reinterpret_cast<uint8_t *>(ws.key + HW_K_CLL);
  uint32_t *clc = ws.key + HW_K_CLC;
  uint32_t *cnt = ws.skey + HW_S_CNT, *nxt = ws.skey + HW_S_NXT;
  {
    const uint32_t cf = lane < 19 ? ws.clf[lane] : 0u;
    const uint32_t bm = __ballot_sync(ZB_FULL, cf != 0);
    const int mc = __popc(bm);
    if (cf) ckey[__popc(bm & lt)] = (cf << 9) | (uint32_t)lane;
    if (lane < 4) ckey[mc + lane] = 0xffffffffu;
    if (lane < 5) reinterpret_cast<uint32_t *>(cll)[lane] = 0;
    __syncwarp();
    if (lane < mc) {
      const uint32_t k = ckey[lane];
      const uint4 *q4 = reinterpret_cast<const uint4 *>(ckey);
      uint32_t r = 0;
      for (int j = 0; j < (mc + 3) >> 2; j++) {
        const uint4 q = q4[j];
        r += (uint32_t)(q.x < k) + (uint32_t)(q.y < k) + (uint32_t)(q.z < k) + (uint32_t)(q.w < k);
      }
      cskey[r] = k;
      ca[r] = k >> 9;
    }
    __syncwarp();
    if (lane == 0) {
      hw_mk(ca, mc, num_c);
      hw_limit(num_c, mc, 7);
    }
    __syncwarp();
    if (lane < mc) cll[cskey[lane] & 511u] = (uint8_t)(mc >= 2 ? hw_len_at(num_c, 7, (uint32_t)lane) : 1u);
    if (lane == 0 && mc < 2) {
      const uint32_t s = mc ? cskey[0] & 511u : 0u;
      cll[s == 0 ? 1 : 0] = 1;
      if (!mc) cll[0] = 1;
    }
    __syncwarp();
    hw_canon(cll, 19, clc, cnt, nxt);
    __syncwarp();
  }
  clk.mark(HWS_CL);

  // ---- block choice and header ----
  // lane i < 19 owns the i-th code-length code length in transmission order (RFC 1951 3.2.7: 16, 17, 18, 0, 8, 7,
  // 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
  const int jo = lane - 3;
  const int ord = lane < 3 ? 16 + lane : jo == 0 ? 0 : (jo & 1) ? 8 + (jo >> 1) : 8 - (jo >> 1);
  const uint32_t ordlen = lane < 19 ? cll[ord] : 0u;
  const int hclen = max(4, (int)__reduce_max_sync(ZB_FULL, ordlen ? (uint32_t)lane + 1u : 0u));
  uint32_t dyn_hdr;
  {
    uint32_t wsum = 0;
    for (int i = lane; i < nr; i += 32) {
      const int sy = rsym[i];
      wsum += cll[sy] + (sy == 16 ? 2u : sy == 17 ? 3u : sy == 18 ? 7u : 0u);
    }
    dyn_hdr = 17u + 3u * (uint32_t)hclen + __reduce_add_sync(ZB_FULL, wsum);
  }
  const uint64_t dyn_bits = dyn_hdr + (uint64_t)dyn_payload + extra;
  const uint64_t fix_bits = 3 + (uint64_t)fix_payload + extra;
  const uint64_t dyn_bytes = is_final ? (dyn_bits + 7) / 8 : (dyn_bits + 3 + 7) / 8 + 4;
  const uint64_t fix_bytes = is_final ? (fix_bits + 7) / 8 : (fix_bits + 3 + 7) / 8 + 4;
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
  uint32_t *tail = ws.skey + HW_S_TAIL, *hdr = tail + 14;
  for (int i = lane; i < HW_TAIL_WORDS - 14; i += 32) hdr[i] = 0;
  __syncwarp();
  uint32_t hdr_bits = 0;
  if (type == 1) {
    if (lane == 0) hdr[0] = is_final | 2u;
    hdr_bits = 3;
    for (int s = lane; s < 320; s += 32) ws.lens[s] = (uint8_t)(s < 288 ? zb_fixed_ll_len(s) : 5);
  } else if (type == 2) {
    if (lane == 0)
      hdr[0] = is_final | 4u | (uint32_t)(nll - 257) << 3 | (uint32_t)(nd - 1) << 8 | (uint32_t)(hclen - 4) << 13;
    __syncwarp();
    if (lane < hclen) hw_or_bits(hdr, 17u + 3u * (uint32_t)lane, ordlen, 3);
    uint32_t pos = 17u + 3u * (uint32_t)hclen;
    for (int base = 0; base < nr; base += 32) {
      const int i = base + lane;
      uint32_t w = 0, v = 0;
      if (i < nr) {
        const int sy = rsym[i];
        const uint32_t cl = cll[sy];
        w = cl + (sy == 16 ? 2u : sy == 17 ? 3u : sy == 18 ? 7u : 0u);
        v = (clc[sy] & 0xffffu) | (uint32_t)rext[i] << cl;
      }
      uint32_t incl = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(ZB_FULL, incl, o);
        if (lane >= o) incl += t;
      }
      if (w) hw_or_bits(hdr, pos + incl - w, v, w);
      pos += __shfl_sync(ZB_FULL, incl, 31);
    }
    hdr_bits = pos;
  }
  __syncwarp();
  clk.mark(HWS_HEADER);

  // ---- canonical codes ----
  if (type == 0) {
    for (int i = lane; i < 320; i += 32) gw[i] = 0;
  } else {
    hw_canon(ws.lens, 288, gw, cnt, nxt);
    hw_canon(ws.lens + 288, 32, gw + 288, cnt, nxt);
  }
  clk.mark(HWS_CODES);

  // ---- per-sub-chunk bit ranges ----
  uint32_t wbs[ZB_WARPS_PER_CHUNK], eob = 0;
#pragma unroll
  for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) wbs[w] = 0;
  if (type != 0) {
    uint32_t part[ZB_WARPS_PER_CHUNK];
#pragma unroll
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) part[w] = 0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
      const int p = lane + 32 * k;
      if (p < ZB_HIST_WORDS) {
        const uint32_t c0 = hw_cost(ws.lens, 2 * p), c1 = hw_cost(ws.lens, 2 * p + 1);
#pragma unroll
        for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
          const uint32_t v = __ldg(hw + w * ZB_HIST_WORDS + p);
          part[w] += (v & 0xffffu) * c0 + (v >> 16) * c1;
        }
      }
    }
    uint32_t pos = hdr_bits;
#pragma unroll
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
      wbs[w] = pos;
      pos += __reduce_add_sync(ZB_FULL, part[w]);
    }
    eob = pos;
  }
  clk.mark(HWS_BITS);

  // ---- store the tail: block_type, hdr_bits, warp_bit_start[8], eob_bit_start, total_bytes, is_final, chunk_len, hdr ----
  if (lane == 0) {
    tail[0] = (uint32_t)type;
    tail[1] = hdr_bits;
#pragma unroll
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) tail[2 + w] = wbs[w];
    tail[10] = eob;
    tail[11] = (uint32_t)best;
    tail[12] = is_final;
    tail[13] = chunk_len;
  }
  __syncwarp();
  for (int i = lane; i < HW_TAIL_WORDS; i += 32) gw[320 + i] = tail[i];
  clk.mark(HWS_STORE);
}

// One warp per chunk, HW_WARPS chunks per CTA.
__global__ void __launch_bounds__(HW_WARPS * 32)
    k_huff(const ZbChunkDesc *__restrict__ desc, const uint16_t *__restrict__ hist, ZbCodebook *__restrict__ cb,
           uint32_t n_chunks, int level, bool fixed_only = false) {
  __shared__ HwWarp ws_all[HW_WARPS];
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t c = blockIdx.x * HW_WARPS + warp;
  if (c >= n_chunks) return;  // the whole warp
  const ZbChunkDesc d = desc[c];
  HwClk clk;
  clk.start();
  hw_build_codebook(ws_all[warp], reinterpret_cast<const uint32_t *>(hist) + (size_t)c * ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS,
                    d.len, (d.flags & ZB_CHUNK_LAST) ? 1u : 0u, level == 0 ? 0 : fixed_only ? 1 : -1, &cb[c], clk);
  clk.publish();
}
