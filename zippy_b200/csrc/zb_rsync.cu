// zb_rsync.cu -- the rsyncable chunk map: content-defined chunk starts (zb200_rsyncable_chunks and the _rsyncable
// compress calls).  The rule is DESIGN.md section 5 "Rsyncable"; tests/native/rsync_model.c restates it:
//  - G[b] (b = 0..255) is the (b + 1)-th output of splitmix64 started from state 0;
//  - h(0) = 0, h(p) = 2 h(p - 1) + G[m[p - 1]] mod 2^64, so h(p) depends on the 64 bytes before p alone;
//  - p is a candidate when 0 < p < L and h(p) >> (64 - ZB_RSYNC_BITS) == 0;
//  - a candidate p is an accepted cut when p >= ZB_RSYNC_MIN and no other candidate lies in (p - MIN, p);
//  - each consecutive pair a < b of {0} + cuts + {L} gives the starts a, a + 64 KiB, a + 128 KiB, ... below b; an
//    empty member has one chunk at 0.
// Two launches:
//  1. k_rsync_cand, one CTA per tile of ZB_RSYNC_MIN bytes: the tile and the 64 bytes in front of it are staged in
//     shared memory, each lane rolls h over its 128 positions after a 64-byte warm-up, and the tile's first and last
//     candidate go to tile_cand.  A tile is MIN bytes long, so any two candidates in it are closer than MIN: only
//     its first can be a cut, and whether it is depends on the last candidate of the tile before it alone (one
//     further back lies more than MIN away).
//  2. k_rsync_starts, one CTA per member: the cut of every tile, then a max-scan (the cut before each) and a
//     sum-scan (the starts each gap contributes) over the member's tiles place the starts.
#include "zb_device.cuh"
#include "zb_kernels.h"

#define RS_TILE ZB_RSYNC_MIN
#define RS_THREADS 128
#define RS_RUN (RS_TILE / RS_THREADS)      // positions a lane checks: 128
#define RS_HALO 64                         // h(p) reads the 64 bytes before p
#define RS_WORDS ((RS_HALO + RS_TILE) / 4)
// shared word g sits at g + g / 32: a lane's run is 32 words, so the lanes of a warp read 32 different banks
#define RS_SLOT(g) ((g) + ((g) >> 5))
#define RS_NONE 0xffffu                    // no candidate (tile offsets are below RS_TILE)
#define RS_STARTS_THREADS 256
#define RS_TILES_PER_THREAD 8

static_assert(RS_RUN % 4 == 0 && RS_RUN / 4 == 32, "a lane's run is one bank-skewed row of 32 words");
static_assert(RS_TILE <= RS_NONE, "tile offsets fit below RS_NONE");

// splitmix64's (b + 1)-th output from state 0: the state has been advanced b + 1 times by the golden gamma
__device__ __forceinline__ uint64_t rs_gear(uint32_t b) {
  uint64_t z = (uint64_t)(b + 1) * 0x9E3779B97F4A7C15ull;
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}

__global__ void __launch_bounds__(RS_THREADS) k_rsync_cand(const uint8_t *__restrict__ src,
                                                           const uint64_t *__restrict__ src_off,
                                                           const uint64_t *__restrict__ tile_off, uint32_t n,
                                                           uint64_t n_tiles, uint32_t *__restrict__ tile_cand) {
  __shared__ uint64_t gear[256];
  __shared__ uint32_t words[RS_SLOT(RS_WORDS) + 1];
  __shared__ uint32_t red[RS_THREADS / 32];
  __shared__ uint32_t member;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t b = tid; b < 256; b += RS_THREADS) gear[b] = rs_gear(b);
  for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    if (tid == 0) {   // the member whose tiles hold t: the last m with tile_off[m] <= t (m < n, tile_off[n] = n_tiles)
      uint32_t lo = 0, hi = n;
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (tile_off[mid] <= t) lo = mid;
        else hi = mid - 1;
      }
      member = lo;
    }
    __syncthreads();
    const uint32_t m = member;
    const uint64_t L = src_off[m + 1] - src_off[m];
    const uint64_t lo = (t - tile_off[m]) * RS_TILE, hi = min(L, lo + RS_TILE);
    // word g holds member positions w0 + 4g .. w0 + 4g + 3, w0 = lo - 64; positions below 0 are never read
    const uint8_t *base = src + src_off[m];
    const uint8_t *end = base + hi;
    const int64_t w0 = (int64_t)lo - RS_HALO;
    const uint32_t g0 = lo == 0 ? RS_HALO / 4 : 0, g1 = (uint32_t)((hi - w0 + 3) / 4);
    // aligned 32-bit loads, shifted into place: every word read holds at least one byte of the member's range
    const uintptr_t a0 = (uintptr_t)(base + w0);
    const uint32_t sh = (uint32_t)(a0 & 3u) * 8u;
    const uint32_t *aw = (const uint32_t *)(a0 & ~(uintptr_t)3);
    for (uint32_t g = g0 + tid; g < g1; g += RS_THREADS) {
      const uint32_t *p = aw + g;
      uint32_t v = __ldg(p);
      if (sh) v = __funnelshift_r(v, (const uint8_t *)(p + 1) < end ? __ldg(p + 1) : 0u, sh);
      words[RS_SLOT(g)] = v;
    }
    __syncthreads();
    uint32_t first = RS_NONE, last = 0;   // last: the offset + 1 of the lane's last candidate, 0 for none
    const uint64_t p0 = lo + (uint64_t)tid * RS_RUN;
    if (p0 < hi) {
      const uint32_t pend = (uint32_t)(min(hi, p0 + RS_RUN) - p0);
      const uint32_t r = tid * (RS_RUN / 4) + RS_HALO / 4;   // the run's first word
      uint64_t h = 0;
      if (p0 > 0)
#pragma unroll 4
        for (uint32_t g = r - RS_HALO / 4; g < r; g++) {
          const uint32_t v = words[RS_SLOT(g)];
#pragma unroll
          for (int b = 0; b < 4; b++) h = (h << 1) + gear[(v >> (8 * b)) & 255u];
        }
      for (uint32_t i = 0; i < pend; i += 4) {
        const uint32_t v = words[RS_SLOT(r + i / 4)];
#pragma unroll
        for (uint32_t b = 0; b < 4; b++) {
          const uint32_t j = i + b;
          if (j < pend) {
            if ((h >> (64 - ZB_RSYNC_BITS)) == 0 && p0 + j > 0) {
              const uint32_t off = (uint32_t)(p0 - lo) + j;
              first = min(first, off);
              last = off + 1;
            }
            h = (h << 1) + gear[(v >> (8 * b)) & 255u];
          }
        }
      }
    }
    first = __reduce_min_sync(0xffffffffu, first);
    last = __reduce_max_sync(0xffffffffu, last);
    if (lane == 0) red[warp] = first | (last << 16);
    __syncthreads();
    if (tid == 0) {
      uint32_t f = RS_NONE, l = 0;
      for (int w = 0; w < RS_THREADS / 32; w++) {
        f = min(f, red[w] & 0xffffu);
        l = max(l, red[w] >> 16);
      }
      tile_cand[t] = f | ((l ? l - 1 : RS_NONE) << 16);
    }
    __syncthreads();   // words, red and member are reused by the next tile
  }
}

// exclusive scan over the CTA, and the CTA's total; op is max or +, both with identity 0; tmp holds one value per warp
template <typename Op>
__device__ __forceinline__ uint64_t rs_block_scan(uint64_t v, Op op, uint64_t *tmp, uint64_t &total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint64_t u = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= (uint32_t)d) v = op(v, u);
  }
  if (lane == 31) tmp[warp] = v;
  v = __shfl_up_sync(0xffffffffu, v, 1);
  if (lane == 0) v = 0;
  __syncthreads();
  if (warp == 0) {
    uint64_t x = lane < RS_STARTS_THREADS / 32 ? tmp[lane] : 0;
#pragma unroll
    for (int d = 1; d < RS_STARTS_THREADS / 32; d <<= 1) {
      const uint64_t u = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= (uint32_t)d) x = op(x, u);
    }
    if (lane < RS_STARTS_THREADS / 32) tmp[lane] = x;
  }
  __syncthreads();
  if (warp > 0) v = op(v, tmp[warp - 1]);
  total = tmp[RS_STARTS_THREADS / 32 - 1];
  __syncthreads();   // tmp is reused by the next scan
  return v;
}

struct RsMax {
  __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a > b ? a : b; }
};
struct RsAdd {
  __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a + b; }
};

__device__ __forceinline__ uint64_t rs_div_up(uint64_t a) { return (a + ZB_CHUNK_BYTES - 1) / ZB_CHUNK_BYTES; }

__global__ void __launch_bounds__(RS_STARTS_THREADS) k_rsync_starts(const uint64_t *__restrict__ src_off,
                                                                    const uint64_t *__restrict__ tile_off,
                                                                    const uint64_t *__restrict__ start_off,
                                                                    const uint32_t *__restrict__ tile_cand, uint32_t n,
                                                                    uint64_t *__restrict__ counts,
                                                                    uint64_t *__restrict__ starts) {
  __shared__ uint64_t tmp[RS_STARTS_THREADS / 32];
  const uint32_t tid = threadIdx.x;
  for (uint32_t m = blockIdx.x; m < n; m += gridDim.x) {
    const uint64_t L = src_off[m + 1] - src_off[m];
    const uint64_t t0 = tile_off[m], nt = tile_off[m + 1] - t0;
    const uint64_t cap = start_off[m + 1] - start_off[m];
    uint64_t *out = starts + start_off[m];
    uint64_t prev_cut = 0, written = 0;   // the last cut so far (0: the member start), starts placed so far
    for (uint64_t k0 = 0; k0 < nt; k0 += (uint64_t)RS_STARTS_THREADS * RS_TILES_PER_THREAD) {
      // this thread's tiles k0 + tid * 8 .. + 7: their cuts (0 for none; a cut is at least MIN > 0)
      uint64_t cut[RS_TILES_PER_THREAD];
      uint64_t mine = 0;
#pragma unroll
      for (int i = 0; i < RS_TILES_PER_THREAD; i++) {
        const uint64_t k = k0 + (uint64_t)tid * RS_TILES_PER_THREAD + i;
        cut[i] = 0;
        if (k < nt) {
          const uint32_t f = tile_cand[t0 + k] & 0xffffu;
          const uint32_t pl = k > 0 ? tile_cand[t0 + k - 1] >> 16 : RS_NONE;
          const uint64_t p = k * RS_TILE + f;
          if (f != RS_NONE && p >= ZB_RSYNC_MIN && (pl == RS_NONE || p - ((k - 1) * RS_TILE + pl) >= ZB_RSYNC_MIN))
            cut[i] = p;
        }
        mine = max(mine, cut[i]);
      }
      // the cut before this thread's first: the last cut of the threads before it, or of the earlier rounds
      uint64_t all_max;
      const uint64_t prev = max(prev_cut, rs_block_scan(mine, RsMax(), tmp, all_max));
      uint64_t cnt = 0, q = prev;
#pragma unroll
      for (int i = 0; i < RS_TILES_PER_THREAD; i++)
        if (cut[i]) {
          cnt += rs_div_up(cut[i] - q);
          q = cut[i];
        }
      uint64_t all_cnt;
      uint64_t at = written + rs_block_scan(cnt, RsAdd(), tmp, all_cnt);
      q = prev;
#pragma unroll
      for (int i = 0; i < RS_TILES_PER_THREAD; i++)
        if (cut[i]) {
          for (uint64_t s = q; s < cut[i]; s += ZB_CHUNK_BYTES, at++)
            if (at < cap) out[at] = s;
          q = cut[i];
        }
      prev_cut = max(prev_cut, all_max);
      written += all_cnt;
    }
    // the last gap, from the last cut to the member end, placed by the whole CTA
    const uint64_t tail = L == 0 ? 1 : rs_div_up(L - prev_cut);
    for (uint64_t j = tid; j < tail; j += RS_STARTS_THREADS)
      if (written + j < cap) out[written + j] = prev_cut + j * ZB_CHUNK_BYTES;
    if (tid == 0) counts[m] = written + tail;
    __syncthreads();   // tmp is reused by the next member
  }
}

cudaError_t zb_launch_rsync(const ZbRsyncWork &w, cudaStream_t s) {
  if (w.n == 0) return cudaSuccess;
  if (w.n_tiles) {
    const unsigned grid = (unsigned)(w.n_tiles < (1u << 30) ? w.n_tiles : (1u << 30));
    k_rsync_cand<<<grid, RS_THREADS, 0, s>>>(w.src, w.src_off, w.tile_off, w.n, w.n_tiles, w.tile_cand);
    if (cudaError_t e = cudaGetLastError()) return e;
  }
  const unsigned grid = (w.n < (1u << 20) ? w.n : (1u << 20));
  k_rsync_starts<<<grid, RS_STARTS_THREADS, 0, s>>>(w.src_off, w.tile_off, w.start_off, w.tile_cand, w.n, w.counts,
                                                    w.starts);
  return cudaGetLastError();
}
