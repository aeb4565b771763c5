// zb_deflate.cu -- the compress pipeline for sm_90a:
//   k_lz    : per-chunk LZ77 parse (one CTA per 64 KiB chunk staged in shared memory by
//             TMA; each warp parses an 8 KiB sub-chunk with a private hash table),
//             fused with the per-sub-chunk symbol histograms and the CRC-32/Adler-32
//             of the chunk.  Replaces encodeSnappy/encodeFragment (snappy.nim:12-163),
//             the histogram side of BlockMetadata (internal.nim:128-131) and the
//             separate crc32/adler32 passes of zippy.nim:47,73.
//   k_huff  : one warp per chunk, four chunks per CTA, workspace in shared memory
//             (zb_huff_warp.cuh): the codebook zb_build_codebook (zb_huff.h) writes, built
//             in parallel stages -- replaces huffmanCodes + the dynamic header writer
//             (deflate.nim:13-151, 295-394) and the stored/fixed/dynamic choice (deflate.nim:274-290).
//   k_scan  : exclusive scan of chunk sizes -> output offsets; per-member checksum combine.
//   k_pack  : token -> bit emission with exact, precomputed bit offsets (replaces the
//             BitStreamWriter loop, deflate.nim:396-464, bitstreams.nim:84-123) plus the
//             gzip/zlib framing bytes of zippy.nim:21-78 for batched members.
#include "zb_device.cuh"
#include "zb_kernels.h"
#include "zb_huff_warp.cuh"

#define LZ_THREADS (ZB_WARPS_PER_CHUNK * 32)
#define LZ_HASH_BITS 11
#define LZ_TABLE_ENTRIES (1 << LZ_HASH_BITS)
#define LZ_PRESEED 2048
#ifndef ZB_LZ1_RESOLVE_WINNER
#define ZB_LZ1_RESOLVE_WINNER 0  // 1: resolve same-entry stores of one instruction in software (deterministic by construction)
#endif
#define LZ_LANE_CAP 32  // bytes a lane extends on its own; a selected match that hit the cap finishes warp-cooperatively

// k_lz walks the chunk in LZ_PHASES phases of 32 KiB: in each phase a warp parses one 4 KiB PIECE with a fresh
// hash table (pre-seeded with the 2 KiB before the piece), so only half the chunk sits in shared memory at a time
// and three CTAs (24 warps) fit on an SM instead of two.  (A full 64 KiB stage + one 8 KiB piece per warp was
// 112 KiB per CTA: 16 warps per SM, too few to hide the parse's latency.  tools/lzsim.c prices the shorter pieces at
// +0.3 % of compressed size.)
#define LZ_PIECE_BYTES ZB_REC_PIECE_BYTES
#define LZ_PHASES (ZB_SUB_BYTES / LZ_PIECE_BYTES)
#define LZ_PHASE_BYTES (ZB_CHUNK_BYTES / LZ_PHASES)
#define LZ_PHASE_HIST 1024  // bytes of the previous phase staged again in front: the pre-seed of the phase's first piece
#define LZ_BATCH_LPW 2      // lanes per window in the batch pass
#define LZ_BATCH_WINDOWS (32 / LZ_BATCH_LPW)
static_assert(LZ_PIECE_BYTES * ZB_WARPS_PER_CHUNK == LZ_PHASE_BYTES, "one piece per warp and phase");
static_assert(LZ_PIECE_BYTES / ZB_WINDOW % LZ_BATCH_WINDOWS == 0, "a batch of windows never straddles two pieces");

// shared-memory layout of k_lz (bytes).  The CRC step table (4 KiB) is loaded by each warp
// into its own hash-table region for the checksum of a piece and overwritten afterwards.
#define LZ_SM_DATA 0
// + 384: match extension reads up to 296 bytes past a piece's end before clamping the length;
// keep those reads inside the data region (they would otherwise race with another warp's table)
#define LZ_SM_DATA_BYTES (LZ_PHASE_BYTES + LZ_PHASE_HIST + 64 + 384)
#define LZ_SM_TABLE (LZ_SM_DATA + LZ_SM_DATA_BYTES)
#define LZ_SM_TABLE_BYTES (ZB_WARPS_PER_CHUNK * LZ_TABLE_ENTRIES * 2)
#define LZ_SM_HIST (LZ_SM_TABLE + LZ_SM_TABLE_BYTES)
#define LZ_SM_HIST_BYTES (ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS * 4)
#define LZ_SM_RING (LZ_SM_HIST + LZ_SM_HIST_BYTES)
#define LZ_SM_RING_BYTES (ZB_WARPS_PER_CHUNK * LZ_BATCH_WINDOWS * ZB_MATCH_SLOTS * 4)
#define LZ_SM_LMUL (LZ_SM_RING + LZ_SM_RING_BYTES)
#define LZ_LMUL_PIECE 33    // lane_mul[33 + k] = x^(8 * 4096 * k), k = 0..15
#define LZ_LMUL_PQ 49       // lane_mul[49 + k] = x^(8 * 1024 * k), k = 0..3
#define LZ_SM_LMUL_BYTES (56 * 4)
#define LZ_SM_PART (LZ_SM_LMUL + LZ_SM_LMUL_BYTES)
#define LZ_SM_PART_BYTES (ZB_WARPS_PER_CHUNK * 24)
#define LZ_SM_BAR (LZ_SM_PART + LZ_SM_PART_BYTES)
#define LZ_SM_TOTAL (LZ_SM_BAR + 16)
static_assert(LZ_TABLE_ENTRIES * 2 >= 4096, "a warp's table region must hold the CRC step table");
static_assert(3 * (LZ_SM_TOTAL + 1024) <= 233472, "three CTAs per SM");
static_assert(LZ_SM_PART % 8 == 0 && LZ_SM_TABLE % 16 == 0, "alignment");

__device__ __forceinline__ uint32_t lz_hash(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - LZ_HASH_BITS); }
// PTX shifts clamp (a shift by >= 32 gives 0), unlike C++ shifts
__device__ __forceinline__ uint32_t shl_clamp(uint32_t x, uint32_t n) {
  uint32_t r;
  asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(n));
  return r;
}
__device__ __forceinline__ uint32_t low_mask(uint32_t n) { return shl_clamp(1u, n) - 1u; }  // n >= 32 -> all ones

// Final match record consumed by k_pack: length code | length extra value << 5 |
// distance code << 10 | distance extra value << 15.
__device__ __forceinline__ uint32_t lz_final_rec(uint32_t mlen, uint32_t dist, int &lc, int &dc) {
  uint32_t le, de;
  lc = (int)zb_len_code_bf(mlen, le);
  dc = (int)zb_dist_code_bf(dist, de);
  return (uint32_t)lc | (le << 5) | ((uint32_t)dc << 10) | (de << 15);
}


// Greedy selection inside one 32-position window, uniform control flow.  Lane i holds the
// match found at position wb + i (m = 0: none; m == LZ_LANE_CAP: at least that long) and its
// distance.  Candidates are followed as a chain "match -> first candidate at or after its
// end" (3 doubling rounds cover the at most 8 matches a window can start); a last match that
// hit the lane cap necessarily leaves the window and is extended by the whole warp, 8 bytes
// per lane.  Position x of the sub-chunk lives at data[off0 + x].
// CAPPED = false: the caller knows that no lane's m reached the lane cap and that no lane below cur has a match;
// then the selection is straight-line code (no exit extension, no test for a window without matches), which lets
// the compiler interleave its chain of warp-wide operations with independent work around it.
template <bool CAPPED = true>
__device__ __forceinline__ void lz_select(const uint8_t *data, uint32_t off0, uint32_t wb, uint32_t b1, uint32_t cur,
                                          uint32_t nvalid, uint32_t &m, uint32_t dist, uint32_t *ring_slot,
                                          uint32_t &sel, uint32_t &ism, uint32_t &endw) {
  const int lane = zb_lane();
  const uint32_t mm = __ballot_sync(ZB_FULL, m != 0);
  endw = 0;
  ism = 0;
  if (!CAPPED || mm) {
    const uint32_t lbit = 1u << lane;
    const uint32_t endp = (uint32_t)lane + m;
    const uint32_t rest = shl_clamp(1u, endp) ? (mm >> endp) : 0u;
    uint32_t nc = rest ? endp + (uint32_t)(__ffs((int)rest) - 1) : 32u;
    uint32_t vis = CAPPED ? 1u << (cur + (uint32_t)(__ffs((int)(mm >> cur)) - 1)) : mm & (0u - mm);
#pragma unroll
    for (int r = 0; r < 3; r++) {
      vis |= __reduce_or_sync(ZB_FULL, (vis & lbit) ? shl_clamp(1u, nc) : 0u);
      const uint32_t t = __shfl_sync(ZB_FULL, nc, (int)(nc & 31u));
      nc = nc < 32u ? t : 32u;
    }
    ism = vis;
    const int lastm = 31 - __clz((int)ism);
    // the coverage before the lane-cap extension: a capped last match covers every position after it whether the
    // extension clips it to the piece or not (the piece end is nvalid, which sel masks), so this reduce need not
    // wait for the extension and runs alongside the shuffle below
    const uint32_t cov = (ism & lbit) ? (low_mask(endp) & ~low_mask((uint32_t)lane)) : 0u;
    const uint32_t covered = __reduce_or_sync(ZB_FULL, cov);
    uint32_t mlast = __shfl_sync(ZB_FULL, m, lastm);
    if (CAPPED && mlast >= LZ_LANE_CAP) {
      const uint32_t md = __shfl_sync(ZB_FULL, dist, lastm);
      const uint32_t pos = wb + (uint32_t)lastm;
      const uint32_t off = off0 + pos + LZ_LANE_CAP + 8u * (uint32_t)lane;
      uint32_t x0 = zb_ld32_unaligned(data, off) ^ zb_ld32_unaligned(data, off - md);
      uint32_t x1 = zb_ld32_unaligned(data, off + 4) ^ zb_ld32_unaligned(data, off + 4 - md);
      uint32_t nm = x0 ? ((uint32_t)(__ffs((int)x0) - 1) >> 3) : 4u + (x1 ? ((uint32_t)(__ffs((int)x1) - 1) >> 3) : 4u);
      uint32_t stop = __ballot_sync(ZB_FULL, nm < 8u);
      if (stop) {
        int first = __ffs((int)stop) - 1;
        mlast = LZ_LANE_CAP + 8u * (uint32_t)first + __shfl_sync(ZB_FULL, nm, first);
      } else {
        mlast = LZ_LANE_CAP + 256u;
      }
      mlast = min(mlast, min((uint32_t)ZB_MAX_MATCH, b1 - pos));
      if (lane == lastm) m = mlast;
    }
    sel = ism | (~covered & ~low_mask(cur) & low_mask(nvalid));
    endw = (CAPPED || ism) ? (uint32_t)lastm + mlast : 0u;  // !CAPPED: ism = 0 when the window has no match
    // rank and record for every lane, so that the store alone is conditional (a predicated store, no branch)
    const uint32_t rank = (uint32_t)__popc(ism & (lbit - 1u));
    const uint32_t rec = (m - 3u) | ((dist - 1u) << 9);
    if (ism & lbit) ring_slot[rank] = rec;
  } else {
    sel = low_mask(nvalid) & ~low_mask(cur);
  }
}

// k_lz<1>'s work on one lane's position p of a window between its probe and its selection, in three steps:
// lz1_probe (the table load and store), lz1_check (the 4-byte check and the first 8-byte extension step, for every
// lane: it needs no entry), lz1_extend (drops a match below entry and extends the others up to the lane cap).
// Position x of the piece lives at data[doff + x].
struct Lz1Lane {
  uint32_t c, lit, m;  // the candidate the probe read, the byte at p, the match length found so far
  uint32_t limit;      // min(258, b1 - p); 0 past the piece end
  uint32_t ip, ic;     // word indices of p and of the compared candidate in data
  uint32_t sp, sc;     // their bit offsets within a word
  uint32_t hp, hc;     // the upper words of the last step, carried into the next one
  bool more;           // the first 12 bytes match: the extension goes on
};

__device__ __forceinline__ void lz1_probe(const uint8_t *data, uint16_t *table, uint32_t doff, uint32_t p,
                                          uint32_t len, Lz1Lane &L, uint32_t &v, bool &can) {
  const uint32_t *w = reinterpret_cast<const uint32_t *>(data);
  L.ip = (doff + p) >> 2;
  L.sp = ((doff + p) & 3u) * 8u;
  L.hp = w[L.ip + 1];  // stays for the check
  v = __funnelshift_r(w[L.ip], L.hp, L.sp);
  L.lit = v & 255u;
  can = p + 4 <= len;
  const uint32_t h = lz_hash(v);
  L.c = table[h];
  __syncwarp();
  // Lanes of this window that share a hash store to the same entry in one instruction:
  // exactly one of them lands, and WHICH is up to the hardware (resolving the winner with
  // __match_any_sync is a large share of the kernel) ...
  if (can) table[h] = (uint16_t)p;
#if ZB_LZ1_RESOLVE_WINNER
  __syncwarp();
  // make the outcome independent of the arbitration: the highest position wins (every round strictly
  // raises the entry, so it ends).  Slows the kernel; off by default because the
  // arbitration IS fixed on this hardware: the lowest lane lands, which tests/test_gpu_lz1_model.py
  // asserts token by token (and this variant's tokens under the highest-position rule)
  for (;;) {
    const bool lost = can && table[h] < (uint16_t)p;
    if (!__any_sync(ZB_FULL, lost)) break;
    if (lost) table[h] = (uint16_t)p;
    __syncwarp();
  }
#endif
}

// Unaligned compare, 8 bytes per step, carrying the upper word of each side: the first step's words are loaded with
// the 4-byte check, so a lane waits for one round of shared-memory loads per 8 bytes.  Branch-free: a lane without a
// candidate in reach compares p with itself, which keeps its loads inside the data region, and has no match.
__device__ __forceinline__ void lz1_check(const uint8_t *data, uint32_t doff, uint32_t p, uint32_t b1,
                                          uint32_t max_dist, uint32_t v, bool can, Lz1Lane &L) {
  const uint32_t *w = reinterpret_cast<const uint32_t *>(data);
  // a match may not cross the piece end (another warp starts its own parse there)
  L.limit = p < b1 ? min((uint32_t)ZB_MAX_MATCH, b1 - p) : 0u;
  const bool ok = can && L.c < p && p - L.c <= max_dist && L.limit >= ZB_MIN_MATCH;
  const uint32_t q = ok ? L.c : p;
  L.ic = (doff + q) >> 2;
  L.sc = ((doff + q) & 3u) * 8u;
  const uint32_t c0 = w[L.ic], hc = w[L.ic + 1];
  const uint32_t np = w[L.ip + 2], nq = w[L.ic + 2], np2 = w[L.ip + 3], nq2 = w[L.ic + 3];
  const uint32_t x = __funnelshift_r(L.hp, np, L.sp) ^ __funnelshift_r(hc, nq, L.sc);
  const uint32_t x2 = __funnelshift_r(np, np2, L.sp) ^ __funnelshift_r(nq, nq2, L.sc);
  const bool hit = ok && __funnelshift_r(c0, hc, L.sc) == v;
  // equal bytes after the first four, up to 8: from the trailing zero bits of x, or of x2 when x is 0 (32 for none)
  const uint32_t tx = __clz((int)__brev(x)), tx2 = __clz((int)__brev(x2));
  const uint32_t eq = (tx + (x ? 0u : tx2)) >> 3;
  L.m = hit ? 4u + eq : 0u;
  L.more = hit && eq == 8u;
  L.hp = np2;
  L.hc = nq2;
}

__device__ __forceinline__ void lz1_extend(const uint8_t *data, bool before_entry, Lz1Lane &L) {
  const uint32_t *w = reinterpret_cast<const uint32_t *>(data);
  if (before_entry) {
    L.m = 0;
  } else if (L.more) {
    uint32_t hp = L.hp, hc = L.hc;
#pragma unroll 1
    for (uint32_t k = 4;; k += 2) {
      const uint32_t np = w[L.ip + k], nq = w[L.ic + k], np2 = w[L.ip + k + 1], nq2 = w[L.ic + k + 1];
      const uint32_t x = __funnelshift_r(hp, np, L.sp) ^ __funnelshift_r(hc, nq, L.sc);
      const uint32_t x2 = __funnelshift_r(np, np2, L.sp) ^ __funnelshift_r(nq, nq2, L.sc);
      if (x) {
        L.m += (uint32_t)(__ffs((int)x) - 1) >> 3;
        break;
      }
      if (k == LZ_LANE_CAP / 4) {
        L.m += 4;
        break;
      }
      if (x2) {
        L.m += 4u + ((uint32_t)(__ffs((int)x2) - 1) >> 3);
        break;
      }
      L.m += 8;
      hp = np2;
      hc = nq2;
    }
  }
  if (L.m < LZ_LANE_CAP) L.m = min(L.m, L.limit);
}

// LPW lanes per window (lane l: window l % (32 / LPW), part l / (32 / LPW)): publish the window's masks, turn
// its raw match records into the packer's records and count every token in the sub-chunk histogram.  The
// records of a 4 KiB piece form one DENSE stream in window order (grecs_piece[rec_base ...]): a prefix sum
// of the windows' match counts places them, and the packer recomputes the same prefix from the masks.
// (Eight fixed slots per window made every record a 4-byte write into its own 32-byte sector: 2.3x the
// algorithmic DRAM traffic.)  The parts of a window split its literals by position and its matches round-robin.
// LITS = false: the caller has counted the literals already (k_lz<1> does it in the window loop, one atomic per
// lane and window instead of a loop here of one LDS + atomic per literal, as long as the busiest part's).
// Matches convert without branches (lz_final_rec).
template <int LPW, bool LITS>
__device__ __forceinline__ void lz_batch_pass(const uint8_t *wdata, bool active, uint32_t ksel, uint32_t kism,
                                              const uint32_t *ring_win, uint32_t *whist, uint2 *gmask_w,
                                              uint32_t *grecs_piece, uint32_t &rec_base) {
  constexpr int NW = 32 / LPW;
  const uint32_t part = (uint32_t)zb_lane() / NW, wi = (uint32_t)zb_lane() % NW;
  if (active && part == 0) *gmask_w = make_uint2(ksel, kism);
  const uint32_t im = active ? kism : 0u;
  const uint32_t pm = (0xffffffffu >> (32 - 32 / LPW)) << (part * (32 / LPW));
  uint32_t s = (LITS && active) ? (ksel & ~kism & pm) : 0u;  // this part's literal tokens
  while (s) {
    const uint32_t bit = (uint32_t)(__ffs((int)s) - 1);
    s &= s - 1;
    const uint32_t sy = wdata[bit];
    atomicAdd(&whist[sy >> 1], 1u << ((sy & 1u) * 16u));
  }
  const uint32_t nmatch = (uint32_t)__popc(im);
  uint32_t incl = nmatch;
#pragma unroll
  for (int o = 1; o < NW; o <<= 1) {
    const uint32_t t = __shfl_up_sync(ZB_FULL, incl, o, NW);
    if (wi >= (uint32_t)o) incl += t;
  }
  uint32_t *grecs_w = grecs_piece + rec_base + incl - nmatch;
  rec_base += __shfl_sync(ZB_FULL, incl, NW - 1);
  for (uint32_t k = part; k < nmatch; k += LPW) {
    const uint32_t raw = ring_win[k];
    int lc, dc;
    const uint32_t fin = lz_final_rec((raw & 511u) + 3u, (raw >> 9) + 1u, lc, dc);
    grecs_w[k] = fin;
    const uint32_t s1 = 257u + (uint32_t)lc, s2 = (uint32_t)ZB_NUM_LITLEN + (uint32_t)dc;
    atomicAdd(&whist[s1 >> 1], 1u << ((s1 & 1u) * 16u));
    atomicAdd(&whist[s2 >> 1], 1u << ((s2 & 1u) * 16u));
  }
}

// -DZB_LZ1_STAGE_CLOCKS=1 (a diagnostic build, never the shipped one; tools/lz1_stages.py makes it): lane 0 of every
// warp of k_lz<1> adds the clock64() cycles of each stage of the parse into zb_lz1_stage_clk, read back (and
// zeroed) by zb200_lz1_stage_clocks.  The stage order is the one LZ1_STAGE_NAMES in that tool prints.
#ifndef ZB_LZ1_STAGE_CLOCKS
#define ZB_LZ1_STAGE_CLOCKS 0
#endif
enum { LZS_WAIT, LZS_CHECKSUM, LZS_SEED, LZS_PROBE, LZS_EXTEND, LZS_SELECT, LZS_BATCH, LZS_BARRIER, LZS_N };
#if ZB_LZ1_STAGE_CLOCKS
__device__ unsigned long long zb_lz1_stage_clk[LZS_N];
#define LZ_CLK_DECL                          \
  unsigned long long clk_acc[LZS_N] = {};    \
  long long clk_t = clock64();
#define LZ_CLK(s)                            \
  if (MODE == 1) {                           \
    const long long clk_n = clock64();       \
    clk_acc[s] += (unsigned long long)(clk_n - clk_t); \
    clk_t = clk_n;                           \
  }
#define LZ_CLK_PUBLISH()                                                                           \
  if (MODE == 1 && lane == 0) {                                                                    \
    _Pragma("unroll") for (int s_ = 0; s_ < LZS_N; s_++) atomicAdd(&zb_lz1_stage_clk[s_], clk_acc[s_]); \
  }
extern "C" int zb200_lz1_stage_clocks(unsigned long long *out) {
  unsigned long long zero[LZS_N] = {};
  if (cudaMemcpyFromSymbol(out, zb_lz1_stage_clk, sizeof(zero)) != cudaSuccess) return -1;
  return cudaMemcpyToSymbol(zb_lz1_stage_clk, zero, sizeof(zero)) == cudaSuccess ? 0 : -1;
}
#else
#define LZ_CLK_DECL
#define LZ_CLK(s)
#define LZ_CLK_PUBLISH()
#endif

// MODE 1: single-probe hash matcher (level 1); 0: literals only (levels 0, -2); 2: the run-length parse
// (ZB200_STRATEGY_RLE): a position is a match of distance 1 when it is not the chunk's first byte and the run of
// bytes equal to the byte before it, cut at the piece end and at 258, is at least 3 long -- zlib's deflate_rle with
// no history across chunk starts and no match across a piece end.  It probes no table.
// CK: the chunk checksums k_member_check reads for the batch's format (ZB_CK_CRC for gzip, ZB_CK_ADLER for
// zlib, 0 for raw DEFLATE); the other fields of chk are left 0.
// max_dist: MODE 1's farthest match (2^window_bits).  Its matches reach at most 4 KiB + 2 KiB back (a piece and its
// pre-seed), so only windows of 4 KiB and less change its parse.
template <int MODE, int CK>
__global__ void __launch_bounds__(LZ_THREADS, 3)
    k_lz(const uint8_t *__restrict__ src, const ZbChunkDesc *__restrict__ desc, uint2 *__restrict__ masks,
         uint32_t *__restrict__ recs, uint16_t *__restrict__ hist, ZbChunkCheck *__restrict__ chk,
         const ZbCrcTables *__restrict__ tabs, uint32_t max_dist) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *data = smem + LZ_SM_DATA;
  uint16_t *table_all = reinterpret_cast<uint16_t *>(smem + LZ_SM_TABLE);
  uint32_t *hist_all = reinterpret_cast<uint32_t *>(smem + LZ_SM_HIST);
  uint32_t *ring_all = reinterpret_cast<uint32_t *>(smem + LZ_SM_RING);
  uint32_t *lane_mul = reinterpret_cast<uint32_t *>(smem + LZ_SM_LMUL);
  uint64_t *part = reinterpret_cast<uint64_t *>(smem + LZ_SM_PART);
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem + LZ_SM_BAR);

  const uint32_t chunk = blockIdx.x;
  const ZbChunkDesc d = desc[chunk];
  const uint32_t len = d.len;
  const int tid = (int)threadIdx.x, lane = tid & 31;
  // tid >> 5, taken through a warp reduction so that the compiler knows it is warp-uniform: then so are every piece
  // bound and the window loop's control flow, and the loop's warp intrinsics need no divergence guards (BRA.DIV)
  const int warp = (int)__reduce_max_sync(ZB_FULL, (uint32_t)tid >> 5);

  if (tid == 0) {
    zb_mbar_init(bar, 1);
    zb_fence_mbar_init();
  }
  __syncthreads();
  const uint32_t mis = (uint32_t)((uintptr_t)(src + d.src_off) & 15u);

  uint16_t *table = table_all + warp * LZ_TABLE_ENTRIES;
  uint32_t *ring = ring_all + warp * LZ_BATCH_WINDOWS * ZB_MATCH_SLOTS;
  uint2 *gmask = masks + (size_t)chunk * ZB_WINDOWS_PER_CHUNK;
  // checksums of this warp's pieces, each already shifted to the end of the chunk (uniform across the warp)
  uint32_t acc_crc = 0;
  uint64_t acc_a = 0, acc_b = 0;
  LZ_CLK_DECL

  for (uint32_t ph = 0; ph < LZ_PHASES; ph++) {
    const uint32_t pbase = ph * LZ_PHASE_BYTES;               // first byte parsed in this phase
    if (ph && pbase >= len) break;
    const uint32_t sbase = ph ? pbase - LZ_PHASE_HIST : 0u;   // first byte staged (a multiple of 16: same misalignment)
    if (ph) __syncthreads();                                  // every warp is done with the previous phase's bytes
    LZ_CLK(LZS_BARRIER)
    if (tid == 0 && len) {
      zb_fence_proxy_async();
      zb_stage_chunk(data, src + d.src_off + sbase, min(len, pbase + LZ_PHASE_BYTES + 384u) - sbase, bar);
    }
    // while the bulk copy is in flight: clear histograms (once), load the CRC tables
    if (CK & ZB_CK_CRC) {
      uint32_t *crc_tab = reinterpret_cast<uint32_t *>(table);
      for (int i = lane; i < 1024; i += 32) crc_tab[i] = (&tabs->mul1024[0][0])[i];
    }
    if (ph == 0) {
      for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS; i += LZ_THREADS) hist_all[i] = 0;
      if (tid < 33) lane_mul[tid] = tabs->lane_mul[tid];
      if (tid >= 64 && tid < 80) lane_mul[LZ_LMUL_PIECE + tid - 64] = tabs->piece_mul[tid - 64];
      if (tid >= 96 && tid < 100) lane_mul[LZ_LMUL_PQ + tid - 96] = tabs->pq_mul[tid - 96];
      __syncthreads();
    } else {
      __syncwarp();
    }
    if (len) zb_mbar_wait(bar, ph & 1u);
    LZ_CLK(LZS_WAIT)

    const uint32_t b0 = pbase + (uint32_t)warp * LZ_PIECE_BYTES;
    if (b0 >= len) continue;
    const uint32_t b1 = min(b0 + LZ_PIECE_BYTES, len);
    const uint32_t doff = mis - sbase;  // chunk position x lives at data[doff + x] (modular: x >= sbase)
    // histograms stay per 8 KiB sub-chunk (k_huff derives the packer warps' bit ranges from them): the two warps
    // whose pieces make up a sub-chunk count into the same one
    uint32_t *whist = hist_all + (b0 / ZB_SUB_BYTES) * ZB_HIST_WORDS;

    // ---- checksums of this piece, shifted to the end of the chunk ----
    if (CK) {
      ZbCheck c = zb_warp_checksums<LZ_PIECE_BYTES, LZ_LMUL_PQ, CK>(data, doff + b0, b1 - b0,
                                                                    reinterpret_cast<const uint32_t *>(table), lane_mul);
      const uint32_t after = len - b1;
      if (after) {
        if (CK & ZB_CK_CRC) {
          const uint32_t shift = ((after & (LZ_PIECE_BYTES - 1)) == 0) ? lane_mul[LZ_LMUL_PIECE + after / LZ_PIECE_BYTES]
                                                                       : zb_xpow8_t(tabs->pow2, after);
          c.crc_raw = zb_gf2_mul(c.crc_raw, shift);
        }
        if (CK & ZB_CK_ADLER) c.b_sum += (uint64_t)after * c.a_sum;
      }
      acc_crc ^= c.crc_raw;
      acc_a += c.a_sum;
      acc_b += c.b_sum;
      __syncwarp();
    }
    LZ_CLK(LZS_CHECKSUM)

    if (MODE == 1) {
      // the table region held the CRC step table until now: empty it
      uint4 ff = make_uint4(~0u, ~0u, ~0u, ~0u);
      uint4 *t4 = reinterpret_cast<uint4 *>(table);
      for (int i = lane; i < LZ_TABLE_ENTRIES * 2 / 16; i += 32) t4[i] = ff;
      __syncwarp();
      // pre-seed the private table with the positions just before this piece (what of them is staged)
      for (uint32_t s = b0 - min((uint32_t)LZ_PRESEED, b0 - sbase); s < b0; s += 32) {
        const uint32_t p = s + (uint32_t)lane;
        const bool can = p + 4 <= len;
        const uint32_t h = lz_hash(zb_ld32_unaligned(data, doff + p));
        if (can) table[h] = (uint16_t)p;
#if ZB_LZ1_RESOLVE_WINNER
        __syncwarp();
        for (;;) {  // same-entry stores of one instruction: the highest position wins (see the main loop)
          const bool lost = can && table[h] < (uint16_t)p;
          if (!__any_sync(ZB_FULL, lost)) break;
          if (lost) table[h] = (uint16_t)p;
          __syncwarp();
        }
#endif
      }
      __syncwarp();
    }
    LZ_CLK(LZS_SEED)
    uint32_t entry = b0;
    uint32_t ksel = 0, kism = 0;  // lanes i and i + 16 keep the masks of window i of the current batch of 16
    uint32_t *grecs = recs + (size_t)chunk * ZB_RECS_PER_CHUNK + (b0 >> 2);  // this piece's record stream
    uint32_t rec_base = 0;
    const uint32_t bl = (uint32_t)lane & (LZ_BATCH_WINDOWS - 1u);
    // the window's masks into this lane's batch slot, and every 16 windows (or at the end) two lanes per window
    // walk its tokens
    auto window_done = [&](uint32_t wb, uint32_t sel, uint32_t ism) {
      const uint32_t win = wb >> 5, slot = win & (LZ_BATCH_WINDOWS - 1u);
      if (bl == slot) {
        ksel = sel;
        kism = ism;
      }
      if (slot == LZ_BATCH_WINDOWS - 1u || wb + 32 >= b1) {
        __syncwarp();
        const uint32_t bwin = win - slot + bl;  // this lane's window
        lz_batch_pass<LZ_BATCH_LPW, MODE == 0>(data + (uint32_t)(doff + (bwin << 5)), bl <= slot, ksel, kism,
                                               ring + bl * ZB_MATCH_SLOTS, whist, gmask + bwin, grecs, rec_base);
        ksel = kism = 0;
        __syncwarp();
      }
      LZ_CLK(LZS_BATCH)
    };
    if (MODE == 1) {
      // A one-window software pipeline.  A window whose lanes all stop below the lane cap ends its last match by
      // wb + 62, so the next window is entered whatever the selection picks: its probe (with its table stores),
      // 4-byte check and first extension step are then exactly the serial parse's, and are issued together with this
      // window's selection, in one basic block; only its lanes below the new entry wait for the selection.  A
      // capped lane (rare), or the piece's last window, drains the pipeline: the next window starts after the
      // selection, as the first one of the piece does and one after skipped windows.
      Lz1Lane L;           // window wb's lane, probed and extended by the previous step when `ahead`
      bool ahead = false;  // warp-uniform
      for (uint32_t wb = b0; wb < b1; wb += 32) {
        uint32_t *ring_win = ring + ((wb >> 5) & (LZ_BATCH_WINDOWS - 1u)) * ZB_MATCH_SLOTS;
        uint32_t sel = 0, ism = 0;
        if (entry < wb + 32) {
          const uint32_t p = wb + (uint32_t)lane;
          const uint32_t nvalid = min(32u, b1 - wb);
          const uint32_t cur = entry - wb;
          uint32_t v, endw;
          bool can;
          if (!ahead) {
            lz1_probe(data, table, doff, p, len, L, v, can);
            LZ_CLK(LZS_PROBE)
            lz1_check(data, doff, p, b1, max_dist, v, can, L);
            lz1_extend(data, p < entry, L);
            LZ_CLK(LZS_EXTEND)
          }
          ahead = wb + 32 < b1 && !__any_sync(ZB_FULL, L.m >= LZ_LANE_CAP);
          if (ahead) {
            Lz1Lane N;
            lz1_probe(data, table, doff, p + 32, len, N, v, can);
            lz1_check(data, doff, p + 32, b1, max_dist, v, can, N);
            lz_select<false>(data, doff, wb, b1, cur, nvalid, L.m, p - L.c, ring_win, sel, ism, endw);
            entry = wb + max(endw, nvalid);
            // the window's literals, one atomic per lane, from the byte the probe already holds
            uint32_t *hw = &whist[L.lit >> 1];
            const uint32_t one = 1u << ((L.lit & 1u) * 16u);
            if ((sel & ~ism) >> lane & 1u) atomicAdd(hw, one);
            LZ_CLK(LZS_SELECT)
            lz1_extend(data, p + 32 < entry, N);
            L = N;
            LZ_CLK(LZS_EXTEND)
          } else {
            lz_select(data, doff, wb, b1, cur, nvalid, L.m, p - L.c, ring_win, sel, ism, endw);
            entry = wb + max(endw, nvalid);
            if ((sel & ~ism) >> lane & 1u) atomicAdd(&whist[L.lit >> 1], 1u << ((L.lit & 1u) * 16u));
            LZ_CLK(LZS_SELECT)
          }
        }
        window_done(wb, sel, ism);
      }
    } else {
      for (uint32_t wb = b0; wb < b1; wb += 32) {
        uint32_t sel = 0, ism = 0;
        if (entry < wb + 32) {
          const uint32_t p = wb + (uint32_t)lane;
          const uint32_t nvalid = min(32u, b1 - wb);
          const uint32_t cur = entry - wb;
          uint32_t m = 0, c = 0, lit = 0;
          if (MODE == 2) {
            // run lengths from one ballot per 32 positions: bit i of eq says byte wb + i equals the byte before it
            // (never at the chunk's first byte); the run at p is the count of consecutive set bits from p, seen 32
            // bytes ahead
            const uint32_t x = doff + p;
            lit = data[x];
            const uint32_t eq0 = __ballot_sync(ZB_FULL, p != 0u && lit == data[x - 1u]);
            const uint32_t eq1 = __ballot_sync(ZB_FULL, data[x + 32u] == data[x + 31u]);
            const uint32_t ahead = __funnelshift_r(eq0, eq1, (uint32_t)lane);  // bits p .. p + 31
            const uint32_t run = ahead == ~0u ? (uint32_t)LZ_LANE_CAP : (uint32_t)(__ffs((int)~ahead) - 1);
            // a run that fills the lane cap is at least that long: lz_select extends it (distance 1) and cuts it there
            const uint32_t limit = p < b1 ? b1 - p : 0u;
            const uint32_t r = run < (uint32_t)LZ_LANE_CAP ? min(run, limit) : run;
            if (p >= entry && r >= 3u && limit >= 3u) m = r;
            c = p - 1u;
          }
          uint32_t endw;
          lz_select(data, doff, wb, b1, cur, nvalid, m, p - c, ring + ((wb >> 5) & (LZ_BATCH_WINDOWS - 1u)) * ZB_MATCH_SLOTS,
                    sel, ism, endw);
          entry = wb + max(endw, nvalid);
          // the run-length parse counts the window's literals here, one atomic per lane
          if (MODE == 2 && ((sel & ~ism) >> lane & 1u)) atomicAdd(&whist[lit >> 1], 1u << ((lit & 1u) * 16u));
          LZ_CLK(LZS_SELECT)
        }
        window_done(wb, sel, ism);
      }
    }
  }
  if (lane == 0) {
    part[warp * 3 + 0] = acc_crc;
    part[warp * 3 + 1] = acc_a;
    part[warp * 3 + 2] = acc_b;
  }
  __syncthreads();
  // ---- publish histograms (packed u16 pairs == the global u16 layout) and chunk checksums ----
  {
    uint32_t *gh = reinterpret_cast<uint32_t *>(hist + (size_t)chunk * ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS);
    for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS; i += LZ_THREADS) gh[i] = hist_all[i];
  }
  LZ_CLK(LZS_BARRIER)
  LZ_CLK_PUBLISH()
  if (tid == 0) {
    uint32_t raw = 0;
    uint64_t a = 0, b = 0;
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
      raw ^= (uint32_t)part[w * 3 + 0];
      a += part[w * 3 + 1];
      b += part[w * 3 + 2];
    }
    ZbChunkCheck cc;
    cc.crc_raw = raw;
    cc.adler = (CK & ZB_CK_ADLER) ? zb_adler_from_sums(a % ZB_ADLER_MOD, b % ZB_ADLER_MOD, len) : 0u;
    chk[chunk] = cc;
  }
}

// ------------------------------------------------------------------------------------
// k_lz2: the matcher for the LZ levels (-1, 2..9; replaces encodeLz77, lz77.nim:10-130, whose
// head/chain arrays -- 256 KiB + 64 KiB per block -- do not fit next to the data).
// Same CTA = chunk / warp = 8 KiB sub-chunk mapping as k_lz; the chunk is staged together with up
// to 32 KiB of the member's preceding bytes so a match can reach back the full DEFLATE window across
// chunk boundaries.  The dictionary is cut into 8 KiB SEGMENTS (= sub-chunks), 16 KiB of u16 positions
// per segment, all in global memory / L2, one set per resident CTA:
//  * phase 1, BUILD: the segments that lie BEFORE some sub-chunk of this chunk (the staged history
//    and all but the last sub-chunk) get a static, direct-mapped table: 8192 entries, entry = the
//    most recent position of the segment with that 13-bit hash.  Plain 2-byte stores, ten
//    instructions per 32 positions, each segment built once.  (The first version gave every warp a
//    private table pre-seeded with its own 32 KiB of history: every position was inserted five times
//    and the tables, five times the size, thrashed the L2 -- most of that kernel was pre-seeding.)
//  * phase 2, PARSE: a warp walks its sub-chunk 32 positions per step; a lane's candidates are the
//    nearest same-hash position inside the window, the four ways of its bucket in the warp's own
//    incremental table (2048 buckets x 4 most recent positions of this sub-chunk so far) and the
//    entry of its hash in each of the four preceding segments' static tables -- nine candidates from
//    five independent loads instead of a dependent chain walk (the reference follows up to `chain`
//    links, lz77.nim:88-109).  Candidates are verified / extended against shared memory nearest first
//    under the level's budget: a level-dependent number of them looked at, at most `maxcand` verified, one
//    more once a match of `good` bytes is in hand (lz77.nim:104 quarters its budget there); the
//    longest wins;
//  * one-step lazy evaluation: a match shorter than `lazy` is dropped when the next position has a
//    longer one (the reference is greedy; this recovers what the bounded search loses).
#define LZ2_HIST 32768
#define LZ2_SEG_BYTES ZB_SUB_BYTES
#define LZ2_SEGS ((ZB_CHUNK_BYTES + LZ2_HIST) / LZ2_SEG_BYTES)     // 12 segments per staged region
#define LZ2_BUCKET_BITS 11
#define LZ2_BUCKETS (1 << LZ2_BUCKET_BITS)                          // per table (own and static)
#define LZ2_TABLES_PER_CTA (ZB_WARPS_PER_CHUNK + LZ2_SEGS)          // 8 own + 12 static
#define LZ2_RING_WINDOWS 8
#define LZ2_SM_DATA_BYTES (ZB_CHUNK_BYTES + LZ2_HIST + 64 + 384)
#define LZ2_SM_HIST (LZ2_SM_DATA_BYTES)
#define LZ2_SM_RING (LZ2_SM_HIST + LZ_SM_HIST_BYTES)
#define LZ2_SM_RING_BYTES (ZB_WARPS_PER_CHUNK * LZ2_RING_WINDOWS * ZB_MATCH_SLOTS * 4)
#define LZ2_SM_CRC (LZ2_SM_RING + LZ2_SM_RING_BYTES)
#define LZ2_SM_LMUL (LZ2_SM_CRC + 4096)
#define LZ2_SM_PART (LZ2_SM_LMUL + LZ_SM_LMUL_BYTES)
#define LZ2_SM_LIST (LZ2_SM_PART + LZ_SM_PART_BYTES)               // verified candidates: 8 x u16 per thread
#define LZ2_SM_BAR (LZ2_SM_LIST + 8 * LZ_THREADS * 2)
#define LZ2_SM_TOTAL (LZ2_SM_BAR + 16)
static_assert(2 * (LZ2_SM_TOTAL + 1024) <= 233472, "two CTAs per SM");

// Resident CTAs per SM, each with its own 20 tables (320 KiB).  One per SM keeps all tables in the H100's 50 MB
// L2 (42 MB on 132 SMs; two per SM: 84 MB): C4 on an H100 SXM at 400 W, 463 ms per 4 GiB against 510 ms with two.
#ifndef LZ2_CTAS_PER_SM
#define LZ2_CTAS_PER_SM 1
#endif
#ifndef LZ2_STATIC_BITS
#define LZ2_STATIC_BITS 13                                          // direct-mapped static tables: 8192 x u16 = one own table's size
#endif
// own bucket = the top 11 bits of the product, static entry = the top 13
__device__ __forceinline__ uint32_t lz2_hash_mul(uint32_t v) { return v * 0x9E3779B1u; }
__device__ __forceinline__ uint32_t lz2_hash(uint32_t v) { return lz2_hash_mul(v) >> (32 - LZ2_BUCKET_BITS); }

// shift `e` into way 0 of a bucket of four u16 entries (most recent first)
__device__ __forceinline__ uint2 lz2_push(uint2 b, uint32_t e) {
  uint2 r;
  r.y = __funnelshift_l(b.x, b.y, 16);
  r.x = (b.x << 16) | (e & 0xffffu);
  return r;
}

__device__ __forceinline__ void lz2_clear_table(uint2 *tab, int bytes = LZ2_BUCKETS * 8) {
  const uint4 ff = make_uint4(~0u, ~0u, ~0u, ~0u);
  uint4 *t4 = reinterpret_cast<uint4 *>(tab);
  for (int i = zb_lane(); i < bytes / 16; i += 32) __stcg(&t4[i], ff);
}

// Insert the window's positions (qwin + lane, for lanes with `can`) into a table in stream order;
// returns each lane's bucket as it was before this window (the lookup) and the mask of lanes
// sharing the lane's hash.  Positions are stored modulo 2^16: a candidate's distance is
// (q - entry) & 0xffff, and since every candidate is verified against the data at that distance
// a stale alias can only cost a compare, never correctness.
__device__ __forceinline__ uint2 lz2_probe_insert(uint2 *tab, uint32_t h, bool can, uint32_t qwin, uint32_t &grp) {
  const int lane = zb_lane();
  grp = __match_any_sync(ZB_FULL, can ? h : (0x80000000u | (uint32_t)lane));
  uint2 old = make_uint2(~0u, ~0u);
  if (can) old = __ldcg(&tab[h]);
  __syncwarp();
  if (can && lane == 31 - __clz((int)grp)) {  // one writer per bucket: pushes every position of the group, in order
    uint2 nb = old;
    for (uint32_t g = grp; g; g &= g - 1) nb = lz2_push(nb, qwin + (uint32_t)(__ffs((int)g) - 1));
    __stcg(&tab[h], nb);
  }
  __syncwarp();
  return old;
}

// Per-position constants of the candidate evaluation.
struct Lz2Pos {
  const uint32_t *data32;  // the staged region as words
  uint32_t poff;           // byte offset of the position in the staged region
  uint32_t q;              // region position (what the tables store, modulo 2^16)
  uint32_t v;              // its four bytes
  uint32_t lim;            // candidates at distance 1..lim are inside the window and the region
  uint32_t limit, stop;    // longest match allowed here; per-lane extension stops at min(limit, lane cap)
};

// Candidate evaluation in two passes, so that the expensive part runs with full lanes:
//  lz2_verify : one candidate (a position modulo 2^16).  Cheap rejection -- the distance test also
//    discards empty entries (0xffff aliases a distance that is out of range, or a real position whose
//    bytes are then compared like any other candidate's) -- then the candidate's four bytes; a survivor's
//    distance is appended to the lane's short list in shared memory.  Every lane runs this for every
//    candidate slot: ~16 instructions, no divergence to speak of.
//  lz2_extend : one list entry.  Extends against shared memory up to the lane cap; the longest match wins,
//    `budget` counts extended candidates (lz77.nim:97-109 counts chain links), a match of `good` bytes
//    leaves room for one more only.  The warp loops over list POSITIONS, so the number of rounds is the
//    longest list of the window (typically 3-5), not the number of slots (9).
#define LZ2_LIST 8
__device__ __forceinline__ void lz2_verify(const Lz2Pos &P, uint32_t e, bool search, uint16_t *dl, uint32_t &n) {
  const uint32_t d = (P.q - e) & 0xffffu;
  if (!search || (d - 1u) >= P.lim) return;
  const uint32_t co = P.poff - d;
  const uint32_t *wc = P.data32 + (co >> 2);
  if (__funnelshift_r(wc[0], wc[1], (co & 3u) * 8u) != P.v) return;
  if (n < LZ2_LIST) dl[n * (uint32_t)LZ_THREADS] = (uint16_t)d;   // entry k of thread t at list[k * LZ_THREADS + t]: conflict-free
  n += n < LZ2_LIST ? 1u : 0u;
}
__device__ __forceinline__ void lz2_extend(const Lz2Pos &P, const uint8_t *data, uint32_t d, uint32_t good, uint32_t &m,
                                           uint32_t &dist, int &budget) {
  const uint32_t co = P.poff - d;
  budget--;
  if (m >= 4 && data[co + m] != data[P.poff + m]) {  // cannot beat the best so far
    if (m >= good && budget > 1) budget = 1;
    return;
  }
  const uint32_t *wc = P.data32 + (co >> 2);
  const uint32_t sc = (co & 3u) * 8u;
  const uint32_t *wp = P.data32 + (P.poff >> 2);
  const uint32_t sp = (P.poff & 3u) * 8u;
  uint32_t hp = wp[1], hc = wc[1];
  uint32_t mc = 4;
#pragma unroll 1
  for (int j = 2; j <= LZ_LANE_CAP / 4; j++) {
    const uint32_t np = wp[j], nq = wc[j];
    const uint32_t x = __funnelshift_r(hp, np, sp) ^ __funnelshift_r(hc, nq, sc);
    if (x) {
      mc += (uint32_t)(__ffs((int)x) - 1) >> 3;
      break;
    }
    mc += 4;
    hp = np;
    hc = nq;
  }
  mc = min(mc, P.limit);  // bytes past the sub-chunk end (another member's, stale shared memory) never count
  if (mc > m) {
    m = mc;
    dist = d;
  }
  if (m >= good && budget > 1) budget = 1;
}

// Stage a ZB_CHUNK_DICT chunk: its hb bytes of history are the end of the dictionary window W, the chunk itself
// comes from src.  The region keeps the layout of zb_stage_chunk(rsrc, hb + len): region position q at
// data[mis + q] with mis = (chunk start - hb) & 15, so the chunk's 16-byte granules start at the aligned offset
// a0 = hb + mis - cmis.  The member's copy of W (ZbMemberDict::wend) ends at an address that is cmis modulo 16, so
// W's tail lines up with the same granules: one bulk copy fills data[0, a0) from W, one fills data[a0, ..) from src
// (with the cmis bytes of src in front of the chunk), and after the wait the <= 15 history bytes at q >= hb - cmis
// are stored from W by plain stores.  Called by thread 0 (the copies) and then by every thread (fix_dict_head).
__device__ __forceinline__ void stage_dict_chunk(uint8_t *data, const uint8_t *chunk, uint32_t len, uint32_t hb,
                                                 const uint8_t *wend, uint64_t *bar) {
  const uint32_t cmis = (uint32_t)((uintptr_t)chunk & 15u);
  const uint32_t mis = (cmis - hb) & 15u, a0 = hb + mis - cmis;
  const uint32_t cbytes = (cmis + len + 15u) & ~15u;
  zb_mbar_expect_tx(bar, a0 + cbytes);
  for (uint32_t done = 0; done < a0;) {
    const uint32_t n = min(a0 - done, 32768u);
    zb_tma_load_1d(data + done, wend - hb - mis + done, n, bar);
    done += n;
  }
  for (uint32_t done = 0; done < cbytes;) {
    const uint32_t n = min(cbytes - done, 32768u);
    zb_tma_load_1d(data + a0 + done, chunk - cmis + done, n, bar);
    done += n;
  }
}
__device__ __forceinline__ void fix_dict_head(uint8_t *data, const uint8_t *chunk, uint32_t hb, const uint8_t *wend) {
  const uint32_t cmis = (uint32_t)((uintptr_t)chunk & 15u);
  const uint32_t mis = (cmis - hb) & 15u;
  const uint32_t q = hb - min(hb, cmis) + threadIdx.x;
  if (q < hb) {
    data[mis + q] = wend[(int)q - (int)hb];
    zb_fence_proxy_async();  // before the next chunk's bulk copies overwrite this byte
  }
}

// MINM: the shortest match kept.  ZB200_STRATEGY_FILTERED instantiates 6: a lane's longest candidate shorter than
// that counts as no match before the lazy rule compares neighbours (zlib deflate_slow's match_length <= 5 rule).
template <bool DICT, int MINM = ZB_MIN_MATCH>
__global__ void __launch_bounds__(LZ_THREADS, 2)
    k_lz2(const uint8_t *__restrict__ src, const ZbChunkDesc *__restrict__ desc, uint2 *__restrict__ masks,
          uint32_t *__restrict__ recs, uint16_t *__restrict__ hist, ZbChunkCheck *__restrict__ chk,
          const ZbCrcTables *__restrict__ tabs, uint2 *__restrict__ tables, uint32_t n_chunks, ZbLz2Params prm,
          const ZbMemberDict *__restrict__ mdict) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *data = smem;
  uint32_t *hist_all = reinterpret_cast<uint32_t *>(smem + LZ2_SM_HIST);
  uint32_t *ring_all = reinterpret_cast<uint32_t *>(smem + LZ2_SM_RING);
  uint32_t *crc_tab = reinterpret_cast<uint32_t *>(smem + LZ2_SM_CRC);
  uint32_t *lane_mul = reinterpret_cast<uint32_t *>(smem + LZ2_SM_LMUL);
  uint64_t *part = reinterpret_cast<uint64_t *>(smem + LZ2_SM_PART);
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem + LZ2_SM_BAR);
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint16_t *dlist = reinterpret_cast<uint16_t *>(smem + LZ2_SM_LIST) + tid;
  uint32_t *whist = hist_all + warp * ZB_HIST_WORDS;
  uint32_t *ring = ring_all + warp * LZ2_RING_WINDOWS * ZB_MATCH_SLOTS;
  uint2 *cta_tabs = tables + (size_t)blockIdx.x * LZ2_TABLES_PER_CTA * LZ2_BUCKETS;
  uint2 *own = cta_tabs + (size_t)warp * LZ2_BUCKETS;              // this warp's incremental table
  uint2 *stat = cta_tabs + (size_t)ZB_WARPS_PER_CHUNK * LZ2_BUCKETS;  // static table of region segment s at stat + s * LZ2_BUCKETS

  if (tid == 0) {
    zb_mbar_init(bar, 1);
    zb_fence_mbar_init();
  }
  for (int i = tid; i < 1024; i += LZ_THREADS) crc_tab[i] = (&tabs->mul1024[0][0])[i];
  if (tid < 33) lane_mul[tid] = tabs->lane_mul[tid];
  if (tid >= 64 && tid < 72) lane_mul[33 + tid - 64] = tabs->sub_mul[tid - 64];
  if (tid >= 96 && tid < 100) lane_mul[41 + tid - 96] = tabs->quart_mul[tid - 96];
  __syncthreads();

  uint32_t phase = 0;
  for (uint32_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    const ZbChunkDesc d = desc[chunk];
    const uint32_t len = d.len, hb = d.pad;  // pad = bytes of history staged in front of the chunk, 0..32768
    // The segment grid is anchored on the chunk start, so the sub-chunks stay segment-aligned: region position q
    // lies in segment (q + hg) / 8192, and only segment 0 is partial when hb is not a multiple of 8 KiB (after a
    // flush).  hg = 0 for every aligned pad.
    const uint32_t hg = (0u - hb) & (LZ2_SEG_BYTES - 1u);
    const uint8_t *rsrc = src + d.src_off - hb;
    const uint32_t mis = (uint32_t)((uintptr_t)rsrc & 15u);
    const uint32_t off0 = mis + hb;           // chunk position x lives at data[off0 + x]
    const uint32_t rlen = hb + len;           // staged bytes; region position q = hb + chunk position
    // DICT: the end of the member's W, in the copy that matches the chunk's alignment
    const uint8_t *wend = DICT && (d.flags & ZB_CHUNK_DICT) ? mdict[d.member].wend : nullptr;
    if (DICT && wend) {
      if (tid == 0) stage_dict_chunk(data, src + d.src_off, len, hb, wend, bar);
    } else if (tid == 0 && rlen) {
      zb_stage_chunk(data, rsrc, rlen, bar);
    }
    for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS; i += LZ_THREADS) hist_all[i] = 0;
    // every table starts empty for every chunk: what a member compresses to does not depend on which
    // chunks this CTA saw before (identical inputs give identical output wherever they sit in a batch)
    lz2_clear_table(own);
    __syncthreads();
    if (rlen) {
      zb_mbar_wait(bar, phase);
      phase ^= 1u;
    }
    if (DICT && wend) {
      fix_dict_head(data, src + d.src_off, hb, wend);
      __syncthreads();
    }

    const uint32_t b0 = (uint32_t)warp * ZB_SUB_BYTES;
    const uint32_t b1 = min(b0 + ZB_SUB_BYTES, len);
    {
      ZbCheck c;
      c.crc_raw = 0;
      c.a_sum = c.b_sum = 0;
      uint32_t n = b0 < len ? b1 - b0 : 0;
      if (n) {
        c = zb_warp_checksums(data, off0 + b0, n, crc_tab, lane_mul);
        const uint32_t after = len - b1;
        if (after) {
          const uint32_t shift = ((after & (ZB_SUB_BYTES - 1)) == 0) ? lane_mul[33 + after / ZB_SUB_BYTES] : zb_xpow8_t(tabs->pow2, after);
          c.crc_raw = zb_gf2_mul(c.crc_raw, shift);
          c.b_sum += (uint64_t)after * c.a_sum;
        }
      }
      if (lane == 0) {
        part[warp * 3 + 0] = c.crc_raw;
        part[warp * 3 + 1] = c.a_sum;
        part[warp * 3 + 2] = c.b_sum;
      }
      __syncwarp();
    }

    // ---- phase 1: static tables of every segment that some sub-chunk of this chunk looks up ----
    {
      const uint32_t nseg = (hg + rlen + LZ2_SEG_BYTES - 1) / LZ2_SEG_BYTES;  // segments of the region; the last is never history
      // the first sub-chunk's segment looks back hist_segs segments (fewer under a small window), the others less far
      const uint32_t seg0 = (hg + hb) / LZ2_SEG_BYTES, sg0 = seg0 > prm.hist_segs ? seg0 - prm.hist_segs : 0u;
      for (uint32_t sg = sg0 + (uint32_t)warp; sg + 1 < nseg; sg += ZB_WARPS_PER_CHUNK) {
        uint2 *tab = stat + (size_t)sg * LZ2_BUCKETS;
        lz2_clear_table(tab, (1 << LZ2_STATIC_BITS) * 2);
        __syncwarp();
        uint16_t *tab16 = reinterpret_cast<uint16_t *>(tab);
        // the segment's region positions [q0, q1): a full segment, but segment 0 starts at the region start
        const uint32_t q0 = sg ? sg * LZ2_SEG_BYTES - hg : 0u, q1 = (sg + 1) * LZ2_SEG_BYTES - hg;
        for (uint32_t s = q0; s < q1; s += 32) {
          const uint32_t q = s + (uint32_t)lane;
          const uint32_t v = zb_ld32_unaligned(data, mis + q);
          const uint32_t hs = lz2_hash_mul(v) >> (32 - LZ2_STATIC_BITS);
          const bool can = q + 4 <= rlen && q < q1;
          // lanes of one window that share a hash would store to one entry in one instruction, and which of
          // them lands is up to the hardware: the highest position writes, the others stand back
          const uint32_t grp = __match_any_sync(ZB_FULL, can ? hs : (0x80000000u | (uint32_t)lane));
          if (can && lane == 31 - __clz((int)grp)) __stcg(&tab16[hs], (uint16_t)q);
        }
        __syncwarp();
      }
    }
    __syncthreads();  // every static table is complete (bar.sync orders the global writes inside the CTA)

    // ---- phase 2: parse ----
    if (b0 < len) {
      const uint32_t myseg = (hg + hb + b0) / LZ2_SEG_BYTES;
      uint32_t entry = b0;
      uint32_t ksel = 0, kism = 0;
      uint2 *gmask = masks + (size_t)chunk * ZB_WINDOWS_PER_CHUNK;
      uint32_t *grecs = recs + (size_t)chunk * ZB_RECS_PER_CHUNK;
      uint32_t rec_base = 0;
      for (uint32_t wb = b0; wb < b1; wb += 32) {
        const uint32_t win = wb >> 5, slot = win & (LZ2_RING_WINDOWS - 1u);
        if ((wb & (ZB_REC_PIECE_BYTES - 1u)) == 0u) rec_base = 0;  // a new 4 KiB piece: its own dense record stream
        const uint32_t p = wb + (uint32_t)lane;
        const uint32_t q = hb + p;               // region position of this lane
        const uint32_t v = zb_ld32_unaligned(data, off0 + p);
        const bool can = (p + 4 <= len);
        const uint32_t h = lz2_hash(v);
        const uint32_t limit = p < b1 ? min((uint32_t)ZB_MAX_MATCH, b1 - p) : 0u;
        const bool search = entry < wb + 32 && can && p >= entry && limit >= ZB_MIN_MATCH;
        // history: the entry of this hash in each of the four preceding segments' tables -- four
        // independent 2-byte loads, in flight while the own table is updated
        const uint32_t hs = lz2_hash_mul(v) >> (32 - LZ2_STATIC_BITS);
        uint32_t hcand[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          hcand[j] = 0xffffu;
          if (search && myseg > (uint32_t)j && prm.hist_segs > (uint32_t)j)
            hcand[j] = __ldcg(reinterpret_cast<const uint16_t *>(stat + (size_t)(myseg - 1u - (uint32_t)j) * LZ2_BUCKETS) + hs);
        }
        uint32_t grp;
        const uint2 bucket = lz2_probe_insert(own, h, can, q - (uint32_t)lane, grp);
        uint32_t sel = 0, ism = 0;
        if (entry < wb + 32) {
          const uint32_t nvalid = min(32u, b1 - wb);
          const uint32_t cur = entry - wb;
          uint32_t m = 0, dist = 1;
          int budget = search ? (int)prm.maxcand : 0;
          Lz2Pos P;
          P.data32 = reinterpret_cast<const uint32_t *>(data);
          P.poff = off0 + p;
          P.q = q;
          P.v = v;
          P.lim = min(q, prm.max_dist);
          P.limit = limit;
          P.stop = min(limit, (uint32_t)LZ_LANE_CAP);
          // candidates, nearest first; the level decides how many are looked at:
          //   the closest same-hash position inside this window
          //   own_ways entries of the own bucket, most recent first
          //   the entries of hist_segs preceding segments, nearest segment first
          uint32_t nl = 0;
          {
            const uint32_t lower = grp & ((1u << lane) - 1u);
            lz2_verify(P, q - ((uint32_t)lane - (uint32_t)(31 - __clz((int)(lower | 1u)))), search && lower != 0u, dlist, nl);
            lz2_verify(P, bucket.x & 0xffffu, search, dlist, nl);
            if (prm.own_ways > 1) lz2_verify(P, bucket.x >> 16, search, dlist, nl);
            if (prm.own_ways > 2) lz2_verify(P, bucket.y & 0xffffu, search, dlist, nl);
            if (prm.own_ways > 3) lz2_verify(P, bucket.y >> 16, search, dlist, nl);
#pragma unroll
            for (int j = 0; j < 4; j++)
              if (prm.hist_segs > (uint32_t)j) lz2_verify(P, hcand[j], search, dlist, nl);
          }
          const uint32_t rounds = __reduce_max_sync(ZB_FULL, nl);
          for (uint32_t k = 0; k < rounds; k++) {
            if (k < nl && budget > 0 && m < P.stop) lz2_extend(P, data, dlist[k * (uint32_t)LZ_THREADS], prm.good, m, dist, budget);
          }
          if (MINM > ZB_MIN_MATCH && m < (uint32_t)MINM) m = 0;
          // one-step lazy evaluation (zlib's max_lazy idea)
          const uint32_t mnext = __shfl_down_sync(ZB_FULL, m, 1);
          if (lane < 31 && m != 0 && m < prm.lazy && mnext > m) m = 0;
          uint32_t endw;
          lz_select(data, off0, wb, b1, cur, nvalid, m, dist, ring + slot * ZB_MATCH_SLOTS, sel, ism, endw);
          entry = wb + max(endw, nvalid);
        }
        const uint32_t bl = (uint32_t)lane & (LZ2_RING_WINDOWS - 1u);
        if (bl == slot) {
          ksel = sel;
          kism = ism;
        }
        if (slot == LZ2_RING_WINDOWS - 1u || wb + 32 >= b1) {
          __syncwarp();
          const uint32_t bwin = win - slot + bl;  // four lanes per window
          lz_batch_pass<32 / LZ2_RING_WINDOWS, true>(data + off0 + (bwin << 5), bl <= slot, ksel, kism, ring + bl * ZB_MATCH_SLOTS,
                                               whist, gmask + bwin,
                                               grecs + ((wb & ~(uint32_t)(ZB_REC_PIECE_BYTES - 1u)) >> 2), rec_base);
          ksel = kism = 0;
          __syncwarp();
        }
      }
    }
    __syncthreads();
    {
      uint32_t *gh = reinterpret_cast<uint32_t *>(hist + (size_t)chunk * ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS);
      for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_WORDS; i += LZ_THREADS) gh[i] = hist_all[i];
    }
    if (tid == 0) {
      uint32_t raw = 0;
      uint64_t a = 0, b = 0;
      for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) {
        raw ^= (uint32_t)part[w * 3 + 0];
        a += part[w * 3 + 1];
        b += part[w * 3 + 2];
      }
      ZbChunkCheck cc;
      cc.crc_raw = raw;
      cc.adler = zb_adler_from_sums(a % ZB_ADLER_MOD, b % ZB_ADLER_MOD, len);
      chk[chunk] = cc;
    }
    __syncthreads();  // shared memory and the CTA's tables are reused by the next chunk
  }
}

// ------------------------------------------------------------------------------------
// k_huff: zb_huff_warp.cuh
#if ZB_HUFF_STAGE_CLOCKS
extern "C" int zb200_huff_stage_clocks(unsigned long long *out) {
  unsigned long long zero[HWS_N] = {};
  if (cudaMemcpyFromSymbol(out, zb_huff_stage_clk, sizeof(zero)) != cudaSuccess) return -1;
  return cudaMemcpyToSymbol(zb_huff_stage_clk, zero, sizeof(zero)) == cudaSuccess ? 0 : -1;
}
#endif

// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t frame_head_bytes(int fmt, const uint8_t *fname_len, uint32_t m,
                                                     const ZbMemberDict *mdict) {
  if (fmt == ZB_DF_GZIP) return 10u + (fname_len ? (uint32_t)fname_len[m] : 0u) + 1u;
  if (fmt == ZB_DF_ZLIB) return mdict && mdict[m].win_len ? 6u : 2u;  // FDICT: DICTID follows CMF / FLG
  return 0u;
}
__device__ __forceinline__ uint32_t frame_tail_bytes(int fmt) {
  return fmt == ZB_DF_GZIP ? 8u : fmt == ZB_DF_ZLIB ? 4u : 0u;
}

#define SCAN_THREADS 1024
__global__ void __launch_bounds__(SCAN_THREADS)
    k_scan(ZbCompressWork w) {
  __shared__ uint64_t warp_tot[32];
  __shared__ uint64_t carry_s;
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry_s = w.out_base_ptr ? *w.out_base_ptr : w.out_base;
  __syncthreads();
  for (uint32_t base = 0; base < w.n_chunks; base += SCAN_THREADS) {
    uint32_t c = base + (uint32_t)tid;
    uint64_t sz = 0;
    uint32_t head = 0, flags = 0, member = 0;
    if (c < w.n_chunks) {
      ZbChunkDesc d = w.desc[c];
      flags = d.flags;
      member = d.member;
      sz = w.cb[c].total_bytes;
      if (flags & ZB_CHUNK_HEAD) {
        head = frame_head_bytes(w.data_format, w.fname_len, member, w.mdict);
        sz += head;
      }
      if (flags & ZB_CHUNK_LAST) sz += frame_tail_bytes(w.data_format);
    }
    uint64_t incl = sz;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t t = __shfl_up_sync(ZB_FULL, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint64_t t = warp_tot[lane], it = t;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint64_t u = __shfl_up_sync(ZB_FULL, it, o);
        if (lane >= o) it += u;
      }
      warp_tot[lane] = it - t;  // exclusive
    }
    __syncthreads();
    uint64_t carry = carry_s;
    uint64_t excl = carry + warp_tot[warp] + incl - sz;
    if (c < w.n_chunks) {
      w.chunk_off[c] = excl + head;
      if (flags & ZB_CHUNK_FIRST) w.member_off[member] = excl;
    }
    __syncthreads();
    if (tid == SCAN_THREADS - 1) carry_s = excl + sz;
    __syncthreads();
  }
  if (tid == 0) w.member_off[w.n_members] = carry_s;
}

// whole-member checksums: one warp per member.  Each lane folds a contiguous run of the member's
// chunks (raw(A||B) = raw(A) * x^(8|B|) + raw(B); Adler by its closed form), then a shuffle tree
// folds the 32 runs, so a member of 16384 chunks (1 GiB) is not combined serially.  A carry-in (the
// member's bytes before this launch) goes in front; the trailer value and ISIZE are of the whole.
__global__ void __launch_bounds__(128)
    k_member_check(ZbCompressWork w) {
  const uint32_t m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (m >= w.n_members) return;  // the whole warp leaves together
  const uint32_t c0 = w.member_first[m], c1 = w.member_first[m + 1];
  const uint32_t per = (c1 - c0 + 31u) / 32u;
  const uint32_t a = min(c1, c0 + lane * per), b = min(c1, a + per);
  uint32_t raw = 0, ad = 1;  // of the empty string
  uint64_t bytes = 0;
  for (uint32_t c = a; c < b; c++) {
    const uint32_t l = w.desc[c].len;
    const ZbChunkCheck cc = w.chk[c];
    if (w.data_format == ZB_DF_ZLIB) ad = zb_adler32_combine(ad, cc.adler, l);
    else if (w.data_format == ZB_DF_GZIP)
      raw = zb_gf2_mul(raw, l == ZB_CHUNK_BYTES ? w.tabs->sub_mul[0] : zb_xpow8_t(w.tabs->pow2, l)) ^ cc.crc_raw;
    bytes += l;
  }
  if (c1 - c0 > 1u) {
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t r_raw = __shfl_down_sync(0xffffffffu, raw, o), r_ad = __shfl_down_sync(0xffffffffu, ad, o);
      const uint64_t r_bytes = __shfl_down_sync(0xffffffffu, bytes, o);
      if ((lane & (uint32_t)(2 * o - 1)) == 0u && r_bytes) {
        if (w.data_format == ZB_DF_ZLIB) ad = zb_adler32_combine(ad, r_ad, r_bytes);
        else if (w.data_format == ZB_DF_GZIP) raw = zb_gf2_mul(raw, zb_xpow8_t(w.tabs->pow2, r_bytes)) ^ r_raw;
        bytes += r_bytes;
      }
    }
  }
  if (lane == 0) {
    if (w.carry_in) {
      const ZbMemberCarry ci = w.carry_in[m];
      if (w.data_format == ZB_DF_ZLIB) ad = zb_adler32_combine(ci.adler, ad, bytes);
      else if (w.data_format == ZB_DF_GZIP) raw = zb_gf2_mul(ci.crc_raw, zb_xpow8_t(w.tabs->pow2, bytes)) ^ raw;
      bytes += ci.bytes;
    }
    if (w.carry_out) {
      ZbMemberCarry co;
      co.crc_raw = raw;
      co.adler = ad;
      co.bytes = bytes;
      w.carry_out[m] = co;
    }
    uint32_t v = 0;
    if (w.data_format == ZB_DF_ZLIB) v = ad;
    else if (w.data_format == ZB_DF_GZIP)
      v = ~(zb_gf2_mul(bytes == ZB_CHUNK_BYTES ? w.tabs->sub_mul[0] : zb_xpow8_t(w.tabs->pow2, bytes), 0xffffffffu) ^ raw);
    w.member_check[m] = v;
    w.member_isize[m] = (uint32_t)bytes;
  }
}

// ------------------------------------------------------------------------------------
// k_index_rec: a compress-time index (ZbIndexWork), one thread per chunk.  A chunk's block starts follow from its
// codebook: a coded block at the chunk's first byte, then (not final) the empty sync block after its end-of-block
// code; or stored pieces of at most 65535 bytes, each 5 header bytes + its bytes.  Output offsets are input
// offsets.  A chunk's output is one part, or two for a 65536-byte stored chunk (65535 + 1: its second piece is a
// block start); the raw CRC-32 of a part is the chunk's (k_lz / k_lz2), or for the two parts derived from it and
// the last byte: raw(A || b) = raw(A) * x^8 + raw(b).
#define IX_XINV8 0x6567cb95u  // x^-8 mod P (reflected): raw(A) = (raw(A || b) + raw(b)) * x^-8

struct IxChunk {
  uint64_t o0, byte0;  // output offset of the chunk's first byte; member byte offset of its first block
  uint32_t len, np;    // input bytes; parts (stored pieces, 1 for a coded block)
  bool sync;           // a coded block that is not final: the sync block follows it
};

__device__ __forceinline__ bool ix_owns(uint64_t lo, uint64_t o) { return (o >> 15) << 15 >= lo; }  // k*32768 in [lo, o]

__global__ void __launch_bounds__(128) k_index_rec(ZbCompressWork w, ZbIndexWork x) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= w.n_chunks) return;
  const uint32_t m = w.desc[c].member, c0 = w.member_first[m], c1 = w.member_first[m + 1];
  const uint64_t obase = w.carry_in ? w.carry_in[m].bytes : 0ull, src0 = w.desc[c0].src_off;
  const uint64_t mbyte = w.member_off[m];
  auto chunk = [&](uint32_t cc) {
    IxChunk k;
    const ZbChunkDesc d = w.desc[cc];
    const ZbCodebook *cb = &w.cb[cc];
    k.o0 = obase + (d.src_off - src0);
    k.byte0 = x.byte_base + w.chunk_off[cc] - mbyte;
    k.len = d.len;
    const bool stored = cb->block_type == 0u;
    k.np = stored && d.len > 65535u ? 2u : 1u;
    k.sync = !stored && !cb->is_final;
    return k;
  };
  // block j of chunk cc: j < np a part's start, j == np the sync block
  auto block = [&](uint32_t cc, const IxChunk &k, uint32_t j, uint64_t &bit) -> uint64_t {
    if (j < k.np) {
      bit = (k.byte0 + (uint64_t)j * 65540ull) * 8ull;
      return k.o0 + (uint64_t)j * 65535ull;
    }
    const ZbCodebook *cb = &w.cb[cc];
    bit = k.byte0 * 8ull + cb->eob_bit_start + (cb->ll[256] >> 16);
    return k.o0 + k.len;
  };
  auto part_raw = [&](uint32_t cc, const IxChunk &k, uint32_t j, uint32_t &plen) -> uint32_t {
    const uint32_t raw = w.chk[cc].crc_raw;
    if (k.np == 1u) {
      plen = k.len;
      return raw;
    }
    const uint32_t rb = zb_crc_raw_byte(0u, w.src[w.desc[cc].src_off + 65535u]);
    plen = j ? 1u : 65535u;
    return j ? rb : zb_gf2_mul(raw ^ rb, IX_XINV8);
  };
  // raw CRC-32 and length of the output from block j of chunk cc up to the next point; closed: the interval ends
  // at that point or at the member's end (false: at the end of a stream launch that does not end the member)
  auto walk = [&](uint32_t cc, uint32_t j, uint64_t &n, bool &closed) -> uint32_t {
    uint32_t raw = 0;
    n = 0;
    IxChunk k = chunk(cc);
    uint64_t lo = 0, bit;
    for (bool first = true;; first = false) {
      const uint64_t o = block(cc, k, j, bit);
      if (!first && ix_owns(lo, o)) {
        closed = true;
        return raw;
      }
      lo = o + 1ull;
      if (j < k.np) {
        uint32_t plen;
        const uint32_t pr = part_raw(cc, k, j, plen);
        raw = zb_gf2_mul(raw, plen == ZB_CHUNK_BYTES ? w.tabs->sub_mul[0] : zb_xpow8_t(w.tabs->pow2, plen)) ^ pr;
        n += plen;
      }
      if (++j < k.np + (k.sync ? 1u : 0u)) continue;
      if (++cc >= c1) {
        closed = (w.desc[c1 - 1].flags & ZB_CHUNK_LAST) != 0u;
        return raw;
      }
      k = chunk(cc);
      j = 0;
    }
  };

  const ZbChunkDesc d = w.desc[c];
  const IxChunk k = chunk(c);
  uint64_t lo;  // the first output offset this chunk's first block start may own
  if (c == c0) {
    lo = (d.flags & ZB_CHUNK_HEAD) ? 0ull : x.lo0;
  } else {
    const IxChunk p = chunk(c - 1);
    lo = (p.sync ? k.o0 : p.o0 + (uint64_t)(p.np - 1u) * 65535ull) + 1ull;
  }
  const uint32_t nb = k.np + (k.sync ? 1u : 0u);
  uint64_t o = 0;
  for (uint32_t j = 0; j < nb; j++) {
    uint64_t bit;
    o = block(c, k, j, bit);
    if (ix_owns(lo, o)) {
      const uint64_t r0 = x.rec_first[m] - x.k0;
      const uint64_t kmin = (lo + 32767ull) >> 15, kmax = o >> 15;
      for (uint64_t kk = kmin; kk <= kmax; kk++) {
        x.rec[2ull * (r0 + kk)] = bit;
        x.rec[2ull * (r0 + kk) + 1ull] = o;
      }
      uint64_t n;
      bool closed;
      const uint32_t raw = walk(c, j, n, closed);
      x.crc[r0 + kmin] = closed ? ~(zb_gf2_mul(zb_xpow8_t(w.tabs->pow2, n), 0xffffffffu) ^ raw) : raw;
    } else if (c == c0 && j == 0u && !(d.flags & ZB_CHUNK_HEAD)) {
      uint64_t n;
      bool closed;
      x.launch_out[1] = walk(c, 0u, n, closed);  // the stream's open interval continues up to the first point
    }
    lo = o + 1ull;
  }
  if (c == w.n_chunks - 1u) x.launch_out[0] = o;
}

// ------------------------------------------------------------------------------------
#define PK_ROW_WORDS 17  // a 32-byte window encodes to at most 32 x 15 bits = 15 words (+ partial)
#define PK_STG_WORDS (PK_ROW_WORDS * 32 + 4)   // one batch of 32 rows + the carried partial word
#define PK_EDGES 10       // piece boundaries of a chunk: header+warp 0, warps 1..7, tail, end
// While a batch's tokens are walked, stg holds only its carried word (stg[0]) and zeros, so the batch's inputs are
// staged there and zeroed again before pk_append: the literal bytes in 36-byte slots, one per window (an odd word
// stride: no bank conflicts when the 32 lanes store or read their own windows; the ninth word absorbs the source's
// misalignment), then the batch's match records (the token loop reads one entry past a window's last record).
#define PK_LIT_OFF 1
#define PK_SLOT_WORDS 9
#define PK_REC_OFF (PK_LIT_OFF + 32 * PK_SLOT_WORDS)
static_assert(PK_REC_OFF + 32 * ZB_MATCH_SLOTS + 1 <= PK_STG_WORDS, "a batch's staged inputs fit in stg");
#define PK_CODE_NONE 320  // codes[] entry of zero bits: the second code of an iteration that has none

// Token -> bits, written with plain coalesced stores (no zero-fill, no global atomics).
// A chunk's stream is a sequence of bit PIECES: [block header + warp 0's tokens], warp 1..7's
// tokens, [end-of-block + byte-aligning tail]; k_huff fixed where each one starts.  A warp turns
// 32 windows at a time into bits -- one LANE per 32-byte window walks the window's tokens and
// concatenates codes into its private row of shared memory; a warp prefix sum of the 32 row
// lengths places the rows -- and ORs the rows into a warp-private staging buffer in shared
// memory that is aligned with the 32-bit words of the output; complete words leave with one
// coalesced store per 32 words, the partial last word is carried into the next batch.  Only the
// words that hold a piece boundary (at most ten per chunk, and the chunk's first and last word,
// which neighbouring chunks / the framing bytes share at byte granularity) are merged in a small
// shared-memory edge table and written at the end, byte-wise where the word leaves the chunk.
struct PkEdges {
  uint32_t word[PK_EDGES];   // relative word index that holds boundary k (sorted)
  uint32_t val[PK_EDGES];
  uint32_t used[PK_EDGES];
};
__device__ __forceinline__ void pk_edge_or(PkEdges *ed, uint32_t relword, uint32_t bits) {
  int k = 0;
#pragma unroll
  for (int i = PK_EDGES - 1; i >= 0; i--)
    if (ed->word[i] == relword) k = i;   // the first boundary in this word owns the slot
  atomicOr(&ed->val[k], bits);
  ed->used[k] = 1u;
}

// One warp: append a batch of rows (lane i: `mybits` bits in rows[k * 32 + i]) at relative bit
// `bitcur`, flush the words that became complete.  stg[0] is relative word sw0.
__device__ __forceinline__ void pk_append(uint32_t *stg, const uint32_t *rows, uint32_t mybits, uint32_t &bitcur,
                                          uint32_t &sw0, uint32_t piece_start, uint32_t *dstw_rel, PkEdges *ed) {
  const int lane = zb_lane();
  uint32_t incl = mybits;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(ZB_FULL, incl, o);
    if (lane >= o) incl += t;
  }
  const uint32_t total = __shfl_sync(ZB_FULL, incl, 31);
  uint32_t pos = bitcur + incl - mybits - sw0 * 32u;   // bit offset of this lane's row inside stg
  for (uint32_t k = 0; k * 32u < mybits; k++) {
    const uint32_t nb = min(32u, mybits - k * 32u);
    uint32_t v = rows[k * 32 + lane];
    if (nb < 32u) v &= (1u << nb) - 1u;
    const uint32_t wi = pos >> 5, sh = pos & 31u;
    atomicOr(&stg[wi], v << sh);
    if (sh && sh + nb > 32u) atomicOr(&stg[wi + 1u], v >> (32u - sh));
    pos += 32u;
  }
  __syncwarp();
  bitcur += total;
  const uint32_t nfull = (bitcur >> 5) - sw0;
  const uint32_t carry = stg[nfull];
  for (uint32_t i = (uint32_t)lane; i < nfull; i += 32) {
    const uint32_t rel = sw0 + i, val = stg[i];
    if (rel * 32u >= piece_start) dstw_rel[rel] = val;   // wholly inside this piece
    else pk_edge_or(ed, rel, val);                        // the piece's first word, shared with its predecessor
    stg[i] = 0u;
  }
  __syncwarp();
  if (lane == 0 && nfull) {
    stg[nfull] = 0u;
    stg[0] = carry;
  }
  sw0 += nfull;
  __syncwarp();
}

// Append the n bits of v to a lane's row (acc: the accn < 32 bits of its incomplete word; accn + n < 64).  The
// low word is stored whether or not it is complete: an incomplete one is stored again when it grows, and the
// row's length leaves out what lies past its end.
__device__ __forceinline__ void pk_put(uint32_t *rows, uint32_t v, uint32_t n, uint32_t &acc, uint32_t &accn,
                                       uint32_t &ri) {
  const uint32_t lo = acc | (v << accn), hi = __funnelshift_l(v, 0u, accn);
  accn += n;
  rows[ri] = lo;
  ri += accn & 32u;  // row word k of lane i is rows[k * 32 + i]
  acc = accn >= 32u ? hi : lo;
  accn &= 31u;
}

__global__ void __launch_bounds__(LZ_THREADS, 6)  // 6 CTAs (48 warps) per SM: <= 40 registers, 36 KiB shared
    k_pack(ZbCompressWork w) {
  // [0,288) litlen, [288,320) dist, [320] none: code | code length << 16 | (code length + extra bits) << 24
  __shared__ uint32_t codes[288 + 32 + 1];
  __shared__ uint32_t rows_all[ZB_WARPS_PER_CHUNK * PK_ROW_WORDS * 32];
  __shared__ uint32_t stg_all[ZB_WARPS_PER_CHUNK * PK_STG_WORDS];
  __shared__ PkEdges ed;

  // a launch group whose output would end beyond the destination is not written at all;
  // the host call then returns DST_TOO_SMALL
  if (w.member_off[w.n_members] > w.dst_cap) return;
  const uint32_t chunk = blockIdx.x;
  const ZbChunkDesc d = w.desc[chunk];
  const ZbCodebook *cb = &w.cb[chunk];
  const uint32_t len = d.len;
  const int tid = (int)threadIdx.x, lane = tid & 31;
  const int warp = (int)__reduce_max_sync(ZB_FULL, (uint32_t)tid >> 5);  // known warp-uniform: see k_lz
  const uint32_t btype = cb->block_type;
  const uint64_t out0 = w.chunk_off[chunk];  // byte offset of this chunk's deflate bytes
  const uint8_t *src = w.src + d.src_off;

  for (int i = tid; i <= PK_CODE_NONE; i += LZ_THREADS) {
    const uint32_t e = i < 288 ? cb->ll[i] : i < 320 ? cb->dd[i - 288] : 0u, clen = e >> 16;
    const uint32_t xb = i > 256 && i < 288 ? zb_len_extra_bits(i - 257) : i >= 288 && i < 320 ? zb_dist_extra_bits(i - 288) : 0;
    codes[i] = (e & 0xffffu) | clen << 16 | (clen + xb) << 24;
  }
  for (int i = tid; i < ZB_WARPS_PER_CHUNK * PK_STG_WORDS; i += LZ_THREADS) stg_all[i] = 0u;

  // ---- framing bytes (zippy.nim:21-42, 50-58, 60-78): every byte written explicitly ----
  if (tid == 32 && (d.flags & ZB_CHUNK_HEAD)) {
    uint8_t *h = w.dst + w.member_off[d.member];
    if (w.data_format == ZB_DF_GZIP) {
      h[0] = 31; h[1] = 139; h[2] = 8; h[3] = 8;  // FNAME flag set, as the reference does
      h[4] = h[5] = h[6] = h[7] = 0;              // MTIME
      h[8] = 0; h[9] = 0;                         // XFL, OS (zippy.nim:22-27 writes zeros)
      uint32_t k = w.fname_len ? w.fname_len[d.member] : 0u;
      for (uint32_t i = 0; i < k; i++) h[10 + i] = (uint8_t)(97 + i);
      h[10 + k] = 0;
    } else if (w.data_format == ZB_DF_ZLIB) {
      // CMF: CM 8, CINFO = window_bits - 8 (0x78 for 32 KiB); FLG: FLEVEL 0 and FCHECK, so that CMF FLG is 31 x k
      const uint32_t cmf = (uint32_t)(__ffs((int)w.max_dist) - 9) << 4 | 8u;
      h[0] = (uint8_t)cmf; h[1] = (uint8_t)((31u - (cmf << 8) % 31u) % 31u);
      if (w.mdict && w.mdict[d.member].win_len) {  // FDICT, FLEVEL 0, FCHECK again, then the DICTID big-endian
        const uint32_t id = w.mdict[d.member].dict_id;
        h[1] = (uint8_t)(0x20u | (31u - ((cmf << 8) | 0x20u) % 31u) % 31u);
        h[2] = (uint8_t)(id >> 24); h[3] = (uint8_t)(id >> 16); h[4] = (uint8_t)(id >> 8); h[5] = (uint8_t)id;
      }
    }
  }
  if (tid == 64 && (d.flags & ZB_CHUNK_LAST)) {
    uint8_t *t = w.dst + out0 + cb->total_bytes;
    uint32_t ck = w.member_check[d.member];
    if (w.data_format == ZB_DF_GZIP) {
      uint32_t isz = w.member_isize[d.member];
      t[0] = (uint8_t)ck; t[1] = (uint8_t)(ck >> 8); t[2] = (uint8_t)(ck >> 16); t[3] = (uint8_t)(ck >> 24);
      t[4] = (uint8_t)isz; t[5] = (uint8_t)(isz >> 8); t[6] = (uint8_t)(isz >> 16); t[7] = (uint8_t)(isz >> 24);
    } else if (w.data_format == ZB_DF_ZLIB) {
      t[0] = (uint8_t)(ck >> 24); t[1] = (uint8_t)(ck >> 16); t[2] = (uint8_t)(ck >> 8); t[3] = (uint8_t)ck;
    }
  }

  if (btype == 0) {
    // stored blocks (deflate.nim:179-205): 1 header byte, LEN, NLEN, bytes
    uint8_t *o = w.dst + out0;
    uint32_t npieces = len == 0 ? 1u : (len + 65534u) / 65535u;
    for (uint32_t pc = 0; pc < npieces; pc++) {
      uint32_t s0 = pc * 65535u, n = min(65535u, len - s0);
      uint8_t *ob = o + (size_t)pc * 5u + s0;
      if (tid == 0) {
        ob[0] = (uint8_t)((cb->is_final && pc == npieces - 1) ? 1 : 0);
        ob[1] = (uint8_t)n; ob[2] = (uint8_t)(n >> 8);
        ob[3] = (uint8_t)~n; ob[4] = (uint8_t)((~n) >> 8);
      }
      for (uint32_t i = (uint32_t)tid; i < n; i += LZ_THREADS) ob[5 + i] = src[s0 + i];
    }
    return;
  }

  // ---- geometry: bits are counted from the 32-bit word that holds the chunk's first byte ----
  const uint64_t gbit0 = out0 * 8ull;
  const uint32_t B0 = (uint32_t)(gbit0 & 31ull);                       // relative bit of the chunk's first bit
  uint32_t *dstw_rel = reinterpret_cast<uint32_t *>(w.dst) + (gbit0 >> 5);  // relative word 0
  const uint32_t end_bit = B0 + cb->total_bytes * 8u;
  if (tid < PK_EDGES) {
    uint32_t b = tid == 0 ? B0 : tid <= 7 ? B0 + cb->warp_bit_start[tid] : tid == 8 ? B0 + cb->eob_bit_start : end_bit;
    ed.word[tid] = b >> 5;
    ed.val[tid] = 0u;
    ed.used[tid] = 0u;
  }
  __syncthreads();

  // ---- this warp's piece ----
  const uint32_t piece_start = warp == 0 ? B0 : B0 + cb->warp_bit_start[warp];
  {
    uint32_t *rows = rows_all + warp * PK_ROW_WORDS * 32;  // word k of lane i at rows[k * 32 + i]
    uint32_t *stg = stg_all + warp * PK_STG_WORDS;
    uint32_t bitcur = piece_start, sw0 = piece_start >> 5;
    if (warp == 0) {
      // block header + dynamic tables: 32 bits per lane and batch
      const uint32_t hb = cb->hdr_bits;
      for (uint32_t base = 0; base < hb; base += 1024u) {
        const uint32_t k = (base >> 5) + (uint32_t)lane;
        uint32_t piece = 0, nb = 0;
        if (k * 32u < hb) {
          for (int j = 0; j < 4; j++) piece |= (uint32_t)cb->hdr[k * 4 + j] << (8 * j);
          nb = min(32u, hb - k * 32u);
        }
        rows[lane] = piece;
        __syncwarp();
        pk_append(stg, rows, nb, bitcur, sw0, piece_start, dstw_rel, &ed);
      }
    }
    const uint32_t b0 = (uint32_t)warp * ZB_SUB_BYTES;
    if (b0 < len) {
      const uint32_t b1 = min(b0 + ZB_SUB_BYTES, len);
      const uint2 *gmask = w.masks + (size_t)chunk * ZB_WINDOWS_PER_CHUNK;
      const uint32_t *grecs = w.recs + (size_t)chunk * ZB_RECS_PER_CHUNK + (size_t)warp * ZB_RECS_PER_SUB;
      const uint32_t nwin = (b1 - b0 + 31u) >> 5;
      const uint32_t mis = (uint32_t)(uintptr_t)(src + b0) & 3u;  // the same for every batch (1 KiB apart)
      uint32_t rec_base = 0;
      for (uint32_t wbase = 0; wbase < nwin; wbase += 32) {
        if (wbase && (wbase & (ZB_REC_PIECE_WINDOWS - 1u)) == 0u) {  // the next 4 KiB piece: its own dense record stream
          grecs += ZB_REC_PIECE_BYTES / 4;
          rec_base = 0;
        }
        const uint32_t widx = wbase + (uint32_t)lane;      // window within the sub-chunk
        const uint32_t win = (b0 >> 5) + widx;              // window within the chunk
        uint2 mk = make_uint2(0u, 0u);
        if (widx < nwin) mk = gmask[win];
        uint32_t s = mk.x;
        const uint32_t im = mk.y;
        // this window's records: dense stream in window order
        const uint32_t nmatch = (uint32_t)__popc(im);
        uint32_t rincl = nmatch;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t t = __shfl_up_sync(ZB_FULL, rincl, o);
          if (lane >= o) rincl += t;
        }
        const uint32_t rtot = __shfl_sync(ZB_FULL, rincl, 31);
        // ---- stage the batch's bytes (from the word that holds its first byte) and records in stg ----
        {
          const uint32_t bbase = b0 + (wbase << 5);
          const uint32_t *pw = reinterpret_cast<const uint32_t *>(src + bbase - mis);
          const uint32_t nword = min(1024u, b1 - bbase) + mis;  // 4 * (words to load) covers this many bytes
          // every load is issued before the first store, so the batch waits for global memory once, not 8 times
          uint32_t v[8];
#pragma unroll
          for (uint32_t j = 0; j < 8; j++) {
            const uint32_t k = (uint32_t)lane + 32u * j;
            v[j] = 4u * k < nword ? __ldg(pw + k) : 0u;
          }
#pragma unroll
          for (uint32_t j = 0; j < 8; j++) {
            const uint32_t k = (uint32_t)lane + 32u * j;
            uint32_t *q = stg + PK_LIT_OFF + k + (k >> 3);  // word k % 8 of slot k / 8
            if (4u * k < nword) *q = v[j];
            if (4u * k < nword && k && (k & 7u) == 0u) q[-1] = v[j];  // and the ninth word of the slot before
          }
          // word 256 (a misaligned source): only the ninth word of the last slot
          if (lane == 0 && 4u * 256u < nword) stg[PK_LIT_OFF + 256 + 32 - 1] = __ldg(pw + 256);
          const uint32_t *brec = grecs + rec_base;
#pragma unroll 4
          for (uint32_t k = (uint32_t)lane; k < rtot; k += 32) stg[PK_REC_OFF + k] = __ldg(brec + k);
        }
        rec_base += rtot;
        __syncwarp();
        // ---- one lane per window: every iteration emits two codes with their extra bits, the same operations
        //      whatever token the lane holds.  A match: length code, distance code.  A literal followed by a
        //      literal: both (the all-literal windows set the warp's iteration count).  A lone literal: it and
        //      the zero-bit code ----
        const uint8_t *lit = reinterpret_cast<const uint8_t *>(stg + PK_LIT_OFF + lane * PK_SLOT_WORDS) + mis;
        uint32_t ri = PK_REC_OFF + rincl - nmatch;  // stg[ri]: the lane's next record
        uint32_t wi = (uint32_t)lane, acc = 0, accn = 0;  // rows[wi]: the lane's incomplete row word
        while (s) {
          const uint32_t t1 = s & (0u - s);
          s ^= t1;
          const uint32_t t2 = s & (0u - s);  // 0: t1 is the last token
          // both bytes are read whatever the tokens are (t2 = 0 reads lit[-1], inside stg): no branch
          const uint32_t l1 = lit[31 - __clz(t1)], l2 = lit[31 - __clz(t2)];
          const uint32_t r = stg[ri];
          const bool is_m = (im & t1) != 0u;
          const bool pair = t2 != 0u && (im & (t1 | t2)) == 0u;
          s ^= pair ? t2 : 0u;
          ri += is_m ? 1u : 0u;
          const uint32_t rec = is_m ? r : 0u;
          const uint32_t sym1 = is_m ? 257u + (rec & 31u) : l1;
          const uint32_t sym2 = is_m ? 288u + ((rec >> 10) & 31u) : pair ? l2 : PK_CODE_NONE;
          const uint32_t e1 = codes[sym1], e2 = codes[sym2];
          pk_put(rows, (e1 & 0xffffu) | ((rec >> 5) & 31u) << __byte_perm(e1, 0u, 0x4442), e1 >> 24, acc, accn, wi);
          pk_put(rows, (e2 & 0xffffu) | (rec >> 15) << __byte_perm(e2, 0u, 0x4442), e2 >> 24, acc, accn, wi);
        }
        rows[wi] = acc;
        __syncwarp();
        for (uint32_t k = (uint32_t)lane; k < PK_REC_OFF - PK_LIT_OFF + rtot; k += 32) stg[PK_LIT_OFF + k] = 0u;
        __syncwarp();
        // wi - lane = 32 x the complete words = their bits
        pk_append(stg, rows, wi - (uint32_t)lane + accn, bitcur, sw0, piece_start, dstw_rel, &ed);
      }
    }
    // the piece's last, partial word (shared with its successor)
    if (lane == 0 && (bitcur & 31u)) pk_edge_or(&ed, sw0, stg[0]);
  }
  // ---- end of block + tail: pad to a byte (final block) or the byte-aligning empty stored block
  //      000 + pad + 00 00 ff ff (more chunks of this member follow) ----
  if (tid == 96) {
    const uint32_t e = codes[256];
    uint32_t pos = B0 + cb->eob_bit_start;
    unsigned long long tv = (unsigned long long)(e & 0xffffu);
    uint32_t nb = e >> 24;
    if (!cb->is_final) {
      nb += 3u;
      nb += (8u - ((pos + nb) & 7u)) & 7u;   // to the byte boundary
      tv |= 0xffff0000ull << nb;
      nb += 32u;
    } else {
      nb += (8u - ((pos + nb) & 7u)) & 7u;
    }
    while (nb) {
      const uint32_t rel = pos >> 5, sh = pos & 31u, take = min(nb, 32u - sh);
      const uint32_t bits = (uint32_t)(tv & ((1ull << take) - 1ull)) << sh;
      if (sh == 0 && take == 32u) dstw_rel[rel] = bits;
      else pk_edge_or(&ed, rel, bits);
      tv >>= take;
      pos += take;
      nb -= take;
    }
  }
  __syncthreads();
  // ---- the words that hold piece boundaries: whole where they lie inside the chunk, byte-wise at its two ends ----
  if (tid < PK_EDGES && ed.used[tid] && (tid == 0 || ed.word[tid] != ed.word[tid - 1])) {
    const uint32_t rel = ed.word[tid], val = ed.val[tid];
    const uint32_t lo = rel * 32u, hi = lo + 32u;
    if (lo >= B0 && hi <= end_bit) dstw_rel[rel] = val;
    else {
      uint8_t *bp = reinterpret_cast<uint8_t *>(dstw_rel + rel);
      for (uint32_t j = 0; j < 4; j++)
        if (lo + 8u * j >= B0 && lo + 8u * j + 8u <= end_bit) bp[j] = (uint8_t)(val >> (8u * j));
    }
  }
}

// ------------------------------------------------------------------------------------
static bool zb_is_lz_level(int level) { return level == -1 || level >= 2; }
// Search effort per level, after the reference's configurationTable (internal.nim:177-189: good / lazy / nice /
// chain per level; lz77.nim:97-109 walks `chain` links and quarters the rest at `good`).  Here the candidates
// come from tables instead of a chain, so the budget is how many candidates are looked at (own_ways of the
// own bucket, the entries of hist_segs preceding segments) and how many of them may pass the 4-byte check
// (maxcand); `good` keeps its meaning and `lazy` is the one-step lazy threshold.  Effort and compressed
// size are monotone in the level.
ZbLz2Params zb_lz2_params(int level, uint32_t max_dist) {
  //                                     own hist maxcand good lazy
  static const ZbLz2Params table[10] = {{4, 4, 4, 8, 16}, {4, 4, 4, 8, 16}, {2, 4, 2, 4, 0},  {2, 4, 3, 4, 6},   {3, 4, 3, 4, 8},
                                        {3, 4, 4, 8, 16}, {4, 4, 4, 8, 16}, {4, 4, 6, 8, 32}, {4, 4, 8, 16, 32}, {4, 4, 8, 32, 64}};
  ZbLz2Params p = table[(level >= 2 && level <= 9) ? level : 6];  // -1 (Default) = level 6
  p.hist_segs = std::min(p.hist_segs, (max_dist + LZ2_SEG_BYTES - 1) / LZ2_SEG_BYTES);
  p.max_dist = max_dist;
  return p;
}
size_t zb_lz2_table_bytes(int *grid_out) {
  int grid = LZ2_CTAS_PER_SM * zb_sm_count();
  if (grid_out) *grid_out = grid;
  return (size_t)grid * LZ2_TABLES_PER_CTA * LZ2_BUCKETS * sizeof(uint2);
}
// the k_lz instance for a level's matcher (MODE) and a format's checksum (CK)
typedef void (*ZbLzKernel)(const uint8_t *, const ZbChunkDesc *, uint2 *, uint32_t *, uint16_t *, ZbChunkCheck *,
                           const ZbCrcTables *, uint32_t);
template <int MODE>
static ZbLzKernel zb_lz_kernel_ck(int ck) {
  return ck == (ZB_CK_CRC | ZB_CK_ADLER) ? k_lz<MODE, ZB_CK_CRC | ZB_CK_ADLER>
         : ck == ZB_CK_CRC               ? k_lz<MODE, ZB_CK_CRC>
         : ck == ZB_CK_ADLER             ? k_lz<MODE, ZB_CK_ADLER>
                                         : k_lz<MODE, 0>;
}
// (index_crc: the raw CRC-32 too, for a compress-time index: zlib takes both checksums, raw DEFLATE gzip's instance)
static ZbLzKernel zb_lz_kernel(int mode, int data_format, bool index_crc = false) {
  int ck = data_format == ZB_DF_GZIP ? ZB_CK_CRC : data_format == ZB_DF_ZLIB ? ZB_CK_ADLER : 0;
  if (index_crc) ck |= ZB_CK_CRC;
  return mode == 2 ? zb_lz_kernel_ck<2>(ck) : mode == 1 ? zb_lz_kernel_ck<1>(ck) : zb_lz_kernel_ck<0>(ck);
}
// function attributes are per device: zb200_init calls this once for the ctx's device
cudaError_t zb_setup_deflate_attrs() {
  cudaError_t e = cudaSuccess;
  static const int fmts[3] = {ZB_DF_GZIP, ZB_DF_ZLIB, ZB_DF_DEFLATE};
  for (int mode = 0; mode < 3; mode++)
    for (int f = 0; f < 4; f++) {
      const ZbLzKernel k = f < 3 ? zb_lz_kernel(mode, fmts[f]) : zb_lz_kernel(mode, ZB_DF_ZLIB, true);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, LZ_SM_TOTAL);
      // three CTAs of 75 KiB: ask for the largest shared-memory carve-out
      if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_lz2<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, LZ2_SM_TOTAL);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_lz2<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, LZ2_SM_TOTAL);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_lz2<false, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, LZ2_SM_TOTAL);
  if (e == cudaSuccess) e = zb_setup_opt_attrs();
  // load the remaining kernels now rather than at their first launch (see zb_setup_inflate_attrs)
  cudaFuncAttributes fa;
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_huff);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_scan);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_member_check);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_pack);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_index_rec);
  return e;
}
cudaError_t zb_launch_lz(const ZbCompressWork &w, cudaStream_t s, bool index_crc) {
  if (w.n_chunks == 0) return cudaSuccess;
  if (w.strategy == ZB_STRATEGY_OPTIMAL) return zb_launch_opt(w, s);
  if (zb_is_lz_level(w.level)) {
    int grid = 0;
    (void)zb_lz2_table_bytes(&grid);
    if ((uint32_t)grid > w.n_chunks) grid = (int)w.n_chunks;
    if (w.strategy == ZB_STRATEGY_FILTERED)
      k_lz2<false, 6><<<grid, LZ_THREADS, LZ2_SM_TOTAL, s>>>(w.src, w.desc, w.masks, w.recs, w.hist, w.chk, w.tabs, w.lz2_tables,
                                                             w.n_chunks, zb_lz2_params(w.level, w.max_dist), nullptr);
    else if (w.dict_hist)
      k_lz2<true><<<grid, LZ_THREADS, LZ2_SM_TOTAL, s>>>(w.src, w.desc, w.masks, w.recs, w.hist, w.chk, w.tabs, w.lz2_tables,
                                                         w.n_chunks, zb_lz2_params(w.level, w.max_dist), w.mdict);
    else
      k_lz2<false><<<grid, LZ_THREADS, LZ2_SM_TOTAL, s>>>(w.src, w.desc, w.masks, w.recs, w.hist, w.chk, w.tabs, w.lz2_tables,
                                                          w.n_chunks, zb_lz2_params(w.level, w.max_dist), nullptr);
  } else {
    const int mode = (w.level == -2 || w.level == 0) ? 0 : w.strategy == ZB_STRATEGY_RLE ? 2 : 1;
    const ZbLzKernel k = zb_lz_kernel(mode, w.data_format, index_crc);
    k<<<w.n_chunks, LZ_THREADS, LZ_SM_TOTAL, s>>>(w.src, w.desc, w.masks, w.recs, w.hist, w.chk, w.tabs, w.max_dist);
  }
  return cudaGetLastError();
}
cudaError_t zb_launch_huff(const ZbCompressWork &w, cudaStream_t s) {
  if (w.n_chunks == 0) return cudaSuccess;
  k_huff<<<(w.n_chunks + HW_WARPS - 1) / HW_WARPS, HW_WARPS * 32, 0, s>>>(w.desc, w.hist, w.cb, w.n_chunks, w.level,
                                                                     w.strategy == ZB_STRATEGY_FIXED);
  return cudaGetLastError();
}
cudaError_t zb_launch_scan(const ZbCompressWork &w, cudaStream_t s) {
  k_scan<<<1, SCAN_THREADS, 0, s>>>(w);
  if (w.n_members) k_member_check<<<(w.n_members + 3) / 4, 128, 0, s>>>(w);  // one warp per member
  return cudaGetLastError();
}
cudaError_t zb_launch_index_rec(const ZbCompressWork &w, const ZbIndexWork &x, cudaStream_t s) {
  if (w.n_chunks == 0) return cudaSuccess;
  k_index_rec<<<(w.n_chunks + 127) / 128, 128, 0, s>>>(w, x);
  return cudaGetLastError();
}
cudaError_t zb_launch_pack(const ZbCompressWork &w, cudaStream_t s) {
  if (w.n_chunks == 0) return cudaSuccess;
  k_pack<<<w.n_chunks, LZ_THREADS, 0, s>>>(w);
  return cudaGetLastError();
}
