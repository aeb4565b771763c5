// zb_optimal.cu -- k_opt: the optimal parse (zb200_compress_batch_optimal and its device / stream forms).
//
// One CTA per 64 KiB chunk (a persistent grid, one CTA per SM), staged with up to 32 KiB of the member's history in
// front exactly as k_lz2 stages it; it writes what k_lz2 writes (masks, the dense per-4 KiB-piece records, the
// per-sub-chunk histograms and the chunk checksums), so k_huff, k_scan and k_pack run unchanged behind it.  The
// rules are DESIGN.md section 4 "k_opt" and tests/native/opt_model.c restates them:
//  1. chains: warp 0 links every region position to the previous one with the same 14-bit hash (at most
//     max_dist back), 32 positions per step, into this CTA's scratch (u16 link distances);
//  2. per round, each warp parses its 8 KiB sub-chunk backwards, 32 positions per step: every lane walks its
//     position's chain (OPT_WALK links, OPT_KEEP hits of four equal bytes, each extended to its full length) and
//     keeps the Pareto set; then the warp runs the shortest-path step for the 32 positions one by one, lanes
//     relaxing 32 match lengths at a time against a 512-entry ring of path costs;
//  3. the path is walked forwards (the token starts of each window follow from the choices), counted into the
//     sub-chunk's histogram; between rounds thread 0 turns the chunk's histogram into code lengths with
//     zb_huff_lengths (the builder k_huff's codebook comes from) and those become the next round's costs.
#include "zb_device.cuh"
#include "zb_kernels.h"

#define OPT_THREADS (ZB_WARPS_PER_CHUNK * 32)
#define OPT_HASH_BITS 14
#define OPT_WALK 16      // chain links a position walks
#define OPT_KEEP 8       // hits (four equal bytes) a walk extends before it stops
#define OPT_ROUNDS 2     // cost rounds: fixed-code costs, then the code lengths of round 1's histogram
#define OPT_UNUSED 13    // bits charged for a symbol the previous round's code leaves without a code
#define OPT_RING 512     // path costs of the positions ahead (a match reaches at most 258 ahead)
#define OPT_REGION (ZB_CHUNK_BYTES + 32768)

// shared memory (bytes)
#define OPT_SM_DATA_BYTES (OPT_REGION + 64 + 384)
#define OPT_SM_HEAD OPT_SM_DATA_BYTES                                      // chain heads, then the per-warp parse state
#define OPT_SM_HEAD_BYTES ((1 << OPT_HASH_BITS) * 4)
#define OPT_WARP_WORDS (OPT_RING + 32 * OPT_KEEP)                         // ring, candidate lists [j][lane]
#define OPT_SM_HIST (OPT_SM_HEAD + OPT_SM_HEAD_BYTES)
#define OPT_SM_HIST_BYTES (ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS * 4)
#define OPT_SM_COST (OPT_SM_HIST + OPT_SM_HIST_BYTES)                     // literal/length costs [286], by length [259], distance codes [30]
#define OPT_SM_COST_BYTES ((ZB_NUM_LITLEN + 2 + 260 + 32) * 4)
#define OPT_SM_CRC (OPT_SM_COST + OPT_SM_COST_BYTES)
#define OPT_SM_LMUL (OPT_SM_CRC + 4096)
#define OPT_SM_PART (OPT_SM_LMUL + 56 * 4)
#define OPT_SM_BAR (OPT_SM_PART + ZB_WARPS_PER_CHUNK * 24)
#define OPT_SM_TOTAL (OPT_SM_BAR + 16)
static_assert(ZB_WARPS_PER_CHUNK * OPT_WARP_WORDS * 4 <= OPT_SM_HEAD_BYTES, "the parse state fits where the chain heads were");
static_assert(OPT_SM_HEAD % 16 == 0 && OPT_SM_PART % 8 == 0, "alignment");
static_assert(OPT_SM_TOTAL + 1024 <= 233472, "one CTA per SM");

__device__ __forceinline__ uint32_t opt_hash(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - OPT_HASH_BITS); }

// Bytes a candidate at region position c shares with region position q, both at data[mis + ...], knowing the first
// four are equal: at most limit.
__device__ __forceinline__ uint32_t opt_extend(const uint8_t *data, uint32_t mis, uint32_t c, uint32_t q, uint32_t limit) {
  uint32_t m = 4;
  while (m < limit) {
    const uint32_t x = zb_ld32_unaligned(data, mis + c + m) ^ zb_ld32_unaligned(data, mis + q + m);
    if (x) {
      m += (uint32_t)(__ffs((int)x) - 1) >> 3;
      break;
    }
    m += 4;
  }
  return min(m, limit);
}

// The code lengths of a chunk histogram (summed over the warps' sub-chunks, one end-of-block) as symbol costs.
__device__ void opt_costs_from_hist(const uint32_t *hist, uint32_t *llc, uint32_t *dcs) {
  uint32_t llf[ZB_NUM_LITLEN], df[ZB_NUM_DIST];
  uint8_t lens[ZB_NUM_LITLEN + ZB_NUM_DIST];
  for (int s = 0; s < ZB_HIST_SYMS; s++) {
    uint32_t t = 0;
    for (int w = 0; w < ZB_WARPS_PER_CHUNK; w++) t += hist[w * ZB_HIST_SYMS + s];
    if (s < ZB_NUM_LITLEN) llf[s] = t;
    else df[s - ZB_NUM_LITLEN] = t;
  }
  llf[256] = 1;
  zb_huff_lengths(llf, ZB_NUM_LITLEN, 15, lens);
  zb_huff_lengths(df, ZB_NUM_DIST, 15, lens + ZB_NUM_LITLEN);
  for (int s = 0; s < ZB_NUM_LITLEN; s++) llc[s] = lens[s] ? lens[s] : OPT_UNUSED;
  for (int s = 0; s < ZB_NUM_DIST; s++) dcs[s] = lens[ZB_NUM_LITLEN + s] ? lens[ZB_NUM_LITLEN + s] : OPT_UNUSED;
}

__global__ void __launch_bounds__(OPT_THREADS, 1)
    k_opt(const uint8_t *__restrict__ src, const ZbChunkDesc *__restrict__ desc, uint2 *__restrict__ masks,
          uint32_t *__restrict__ recs, uint16_t *__restrict__ hist, ZbChunkCheck *__restrict__ chk,
          const ZbCrcTables *__restrict__ tabs, uint16_t *__restrict__ links_all, uint32_t *__restrict__ choice_all,
          uint32_t n_chunks, uint32_t max_dist) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t *data = smem;
  uint32_t *head = reinterpret_cast<uint32_t *>(smem + OPT_SM_HEAD);
  uint32_t *hist_all = reinterpret_cast<uint32_t *>(smem + OPT_SM_HIST);
  uint32_t *llc = reinterpret_cast<uint32_t *>(smem + OPT_SM_COST);   // symbol costs, literal/length
  uint32_t *lcost = llc + ZB_NUM_LITLEN + 2;                           // length symbol + extra bits, by length
  uint32_t *dcost = lcost + 260;                                       // distance symbol + extra bits, by code
  uint32_t *crc_tab = reinterpret_cast<uint32_t *>(smem + OPT_SM_CRC);
  uint32_t *lane_mul = reinterpret_cast<uint32_t *>(smem + OPT_SM_LMUL);
  uint64_t *part = reinterpret_cast<uint64_t *>(smem + OPT_SM_PART);
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem + OPT_SM_BAR);
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t *ring = head + warp * OPT_WARP_WORDS;   // after the chains are built
  uint32_t *cand = ring + OPT_RING;                // entry j of lane l at cand[j * 32 + l]: length << 16 | distance
  uint32_t *whist = hist_all + warp * ZB_HIST_SYMS;
  uint16_t *links = links_all + (size_t)blockIdx.x * OPT_REGION;
  uint32_t *choice = choice_all + (size_t)blockIdx.x * ZB_CHUNK_BYTES;

  if (tid == 0) {
    zb_mbar_init(bar, 1);
    zb_fence_mbar_init();
  }
  for (int i = tid; i < 1024; i += OPT_THREADS) crc_tab[i] = (&tabs->mul1024[0][0])[i];
  if (tid < 33) lane_mul[tid] = tabs->lane_mul[tid];
  if (tid >= 64 && tid < 72) lane_mul[33 + tid - 64] = tabs->sub_mul[tid - 64];
  if (tid >= 96 && tid < 100) lane_mul[41 + tid - 96] = tabs->quart_mul[tid - 96];
  __syncthreads();

  uint32_t phase = 0;
  for (uint32_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    const ZbChunkDesc d = desc[chunk];
    const uint32_t len = d.len, hb = d.pad;
    const uint8_t *rsrc = src + d.src_off - hb;
    const uint32_t mis = (uint32_t)((uintptr_t)rsrc & 15u);
    const uint32_t off0 = mis + hb;  // chunk position p at data[off0 + p]
    const uint32_t rlen = hb + len;
    if (tid == 0 && rlen) zb_stage_chunk(data, rsrc, rlen, bar);
    for (int i = tid; i < (1 << OPT_HASH_BITS); i += OPT_THREADS) head[i] = ~0u;
    __syncthreads();
    if (rlen) {
      zb_mbar_wait(bar, phase);
      phase ^= 1u;
    }

    const uint32_t b0 = (uint32_t)warp * ZB_SUB_BYTES;
    const uint32_t b1 = min(b0 + ZB_SUB_BYTES, len);
    {
      ZbCheck c;
      c.crc_raw = 0;
      c.a_sum = c.b_sum = 0;
      if (b0 < len) {
        c = zb_warp_checksums(data, off0 + b0, b1 - b0, crc_tab, lane_mul);
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
    }

    // ---- 1. chains: link[q] = distance to the previous region position with q's hash, 0 for none or too far ----
    if (warp == 0) {
      for (uint32_t s = 0; s < rlen; s += 32) {
        const uint32_t q = s + (uint32_t)lane;
        const bool can = q + 4 <= rlen;
        const uint32_t h = can ? opt_hash(zb_ld32_unaligned(data, mis + q)) : 0u;
        const uint32_t grp = __match_any_sync(ZB_FULL, can ? h : (0x80000000u | (uint32_t)lane));
        const uint32_t lower = grp & ((1u << lane) - 1u);
        const uint32_t prev = lower ? s + (uint32_t)(31 - __clz((int)lower)) : (can ? head[h] : ~0u);
        __syncwarp();
        if (can && lane == 31 - __clz((int)grp)) head[h] = q;
        if (q < rlen) __stcg(&links[q], (uint16_t)(can && prev != ~0u && q - prev <= max_dist ? q - prev : 0u));
        __syncwarp();
      }
    }
    for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS; i += OPT_THREADS) hist_all[i] = 0;
    for (int i = tid; i < ZB_NUM_LITLEN; i += OPT_THREADS) llc[i] = (uint32_t)zb_fixed_ll_len(i);
    if (tid < ZB_NUM_DIST) dcost[tid] = 5u;
    __syncthreads();

    for (int round = 0; round < OPT_ROUNDS; round++) {
      const bool last = round == OPT_ROUNDS - 1;
      for (uint32_t L = (uint32_t)tid + ZB_MIN_MATCH; L <= ZB_MAX_MATCH; L += OPT_THREADS) {
        const int c = zb_len_code(L);
        lcost[L] = llc[257 + c] + (uint32_t)zb_len_extra_bits(c);
      }
      __syncthreads();
      if (tid < ZB_NUM_DIST) dcost[tid] += (uint32_t)zb_dist_extra_bits(tid);
      __syncthreads();

      if (b0 < len) {
        // ---- 2. backwards: candidates of 32 positions, then their shortest-path steps, last position first ----
        if (lane == 0) ring[b1 & (OPT_RING - 1)] = 0u;
        for (uint32_t wb = b0 + ((b1 - 1 - b0) & ~31u);; wb -= 32) {
          const uint32_t p = wb + (uint32_t)lane;
          uint32_t nc = 0;
          {
            const uint32_t limit = p < b1 ? min((uint32_t)ZB_MAX_MATCH, b1 - p) : 0u;
            if (limit >= ZB_MIN_MATCH) {
              const uint32_t q = hb + p, v = zb_ld32_unaligned(data, mis + q);
              uint32_t c = q, best = 0, hits = 0;
              for (int link = 0; link < OPT_WALK; link++) {
                const uint32_t step = __ldcg(&links[c]);
                if (step == 0) break;
                c -= step;
                const uint32_t dd = q - c;
                if (dd > max_dist) break;
                if (zb_ld32_unaligned(data, mis + c) != v) continue;
                hits++;
                const uint32_t m = opt_extend(data, mis, c, q, limit);
                if (m > best) {
                  best = m;
                  cand[nc * 32 + (uint32_t)lane] = m << 16 | dd;
                  nc++;
                }
                if (hits == OPT_KEEP || best == limit) break;
              }
            }
          }
          __syncwarp();
          uint32_t mych = 0;
          for (int i = 31; i >= 0; i--) {
            const uint32_t pi = wb + (uint32_t)i;
            const uint32_t n = __shfl_sync(ZB_FULL, nc, i);
            if (pi >= b1) continue;
            uint32_t best = (llc[data[off0 + pi]] + ring[(pi + 1) & (OPT_RING - 1)]) << 9 | 1u;
            if (n) {
              const uint32_t maxlen = cand[(n - 1) * 32 + (uint32_t)i] >> 16;
              for (uint32_t L0 = ZB_MIN_MATCH; L0 <= maxlen; L0 += 32) {
                const uint32_t L = L0 + (uint32_t)lane;
                if (L <= maxlen) {
                  uint32_t j = 0, e = cand[i];
                  while ((e >> 16) < L) e = cand[++j * 32 + (uint32_t)i];
                  const uint32_t key = (lcost[L] + dcost[zb_dist_code(e & 0xffffu)] + ring[(pi + L) & (OPT_RING - 1)]) << 9 | L;
                  best = min(best, key);
                }
              }
              best = __reduce_min_sync(ZB_FULL, best);
            }
            const uint32_t L = best & 511u;
            uint32_t dist = 0;
            if (L > 1) {
              uint32_t j = 0, e = cand[i];
              while ((e >> 16) < L) e = cand[++j * 32 + (uint32_t)i];
              dist = e & 0xffffu;
            }
            __syncwarp();
            if (lane == 0) ring[pi & (OPT_RING - 1)] = best >> 9;
            if (lane == i) mych = L << 16 | dist;
            __syncwarp();
          }
          if (p < b1) __stcg(&choice[p], mych);
          if (wb == b0) break;
        }
        __syncwarp();

        // ---- 3. forwards: the path's token starts per window, its histogram, and in the last round its masks and records ----
        uint2 *gmask = masks + (size_t)chunk * ZB_WINDOWS_PER_CHUNK;
        uint32_t *grecs = recs + (size_t)chunk * ZB_RECS_PER_CHUNK;
        uint32_t cur = 0, rec_base = 0;
        for (uint32_t wb = b0; wb < b1; wb += 32) {
          if ((wb & (ZB_REC_PIECE_BYTES - 1u)) == 0u) rec_base = 0;
          const uint32_t p = wb + (uint32_t)lane, nvalid = min(32u, b1 - wb);
          const uint32_t ch = p < b1 ? __ldcg(&choice[p]) : (1u << 16);
          const uint32_t myL = ch >> 16;
          uint32_t t = cur, sel = 0, ism = 0;
          while (t < nvalid) {
            const uint32_t Lt = __shfl_sync(ZB_FULL, myL, (int)t);
            sel |= 1u << t;
            if (Lt > 1) ism |= 1u << t;
            t += Lt;
          }
          cur = t - 32u;  // (a path ends exactly at b1, so only full windows carry on)
          const uint32_t lbit = 1u << lane;
          if (sel & lbit) {
            if (myL == 1) {
              atomicAdd(&whist[data[off0 + p]], 1u);
            } else {
              uint32_t le, de;
              const uint32_t lc = zb_len_code_bf(myL, le), dc = zb_dist_code_bf(ch & 0xffffu, de);
              atomicAdd(&whist[257 + lc], 1u);
              atomicAdd(&whist[ZB_NUM_LITLEN + dc], 1u);
              if (last)
                grecs[((wb & ~(uint32_t)(ZB_REC_PIECE_BYTES - 1u)) >> 2) + rec_base + (uint32_t)__popc(ism & (lbit - 1u))] =
                    lc | (le << 5) | (dc << 10) | (de << 15);
            }
          }
          if (last && lane == 0) gmask[wb >> 5] = make_uint2(sel, ism);
          rec_base += (uint32_t)__popc(ism);
        }
      }
      __syncthreads();
      if (!last) {
        if (tid == 0) opt_costs_from_hist(hist_all, llc, dcost);
        __syncthreads();
        for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS; i += OPT_THREADS) hist_all[i] = 0;
      }
    }

    {
      uint16_t *gh = hist + (size_t)chunk * ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS;
      for (int i = tid; i < ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS; i += OPT_THREADS) gh[i] = (uint16_t)hist_all[i];
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
    __syncthreads();  // shared memory and the CTA's scratch are reused by the next chunk
  }
}

size_t zb_opt_scratch_bytes(int *grid_out) {
  const int grid = zb_sm_count();
  if (grid_out) *grid_out = grid;
  return (size_t)grid * (OPT_REGION * sizeof(uint16_t) + ZB_CHUNK_BYTES * sizeof(uint32_t));
}

cudaError_t zb_setup_opt_attrs() {
  return cudaFuncSetAttribute(k_opt, cudaFuncAttributeMaxDynamicSharedMemorySize, OPT_SM_TOTAL);
}

cudaError_t zb_launch_opt(const ZbCompressWork &w, cudaStream_t s) {
  if (w.n_chunks == 0) return cudaSuccess;
  int grid = 0;
  (void)zb_opt_scratch_bytes(&grid);
  if ((uint32_t)grid > w.n_chunks) grid = (int)w.n_chunks;
  uint16_t *links = reinterpret_cast<uint16_t *>(w.opt_scratch);
  uint32_t *choice = reinterpret_cast<uint32_t *>(w.opt_scratch + (size_t)grid * OPT_REGION * sizeof(uint16_t));
  k_opt<<<grid, OPT_THREADS, OPT_SM_TOTAL, s>>>(w.src, w.desc, w.masks, w.recs, w.hist, w.chk, w.tabs, links, choice,
                                                 w.n_chunks, w.max_dist);
  return cudaGetLastError();
}
