// zb_device.cuh -- device-side helpers shared by the sm_90a kernels:
// TMA 1-D bulk staging + mbarrier, unaligned shared-memory reads, the warp-level
// lane-strided CRC-32 / Adler-32 body (algebra in zb_crc.h, CPU-checked in
// tests/test_host_units.py::test_crc_math).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "zb_common.h"
#include "zb_crc.h"

#define ZB_FULL 0xffffffffu

// SMs of the current device (grid sizes of the persistent and grid-stride kernels); 132 on an H100 SXM
static inline int zb_sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

__device__ __forceinline__ uint32_t zb_smem_addr(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ int zb_lane() { return (int)(threadIdx.x & 31u); }

// ---- mbarrier + TMA bulk copy (cp.async.bulk -> SASS UBLKCP) ----
__device__ __forceinline__ void zb_mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(zb_smem_addr(bar)), "r"(count) : "memory");
}
// orders this thread's earlier generic-proxy accesses of shared memory before its later async-proxy (bulk copy) ones
__device__ __forceinline__ void zb_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void zb_fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void zb_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(zb_smem_addr(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void zb_mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(zb_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void zb_mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "ZB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra ZB_DONE_%=;\n"
      "bra ZB_WAIT_%=;\n"
      "ZB_DONE_%=:\n"
      "}\n" ::"r"(zb_smem_addr(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy; src, dst 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void zb_tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                               uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          zb_smem_addr(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(zb_smem_addr(bar))
      : "memory");
}

// Stage `len` bytes starting at global `src` (any alignment) into `buf` so that byte i
// of the input lives at buf[mis + i], mis = src & 15.  buf must be 16-byte aligned and
// hold round_up(mis + len, 16) bytes.  Called by one thread; everyone then waits on bar.
// Reads up to 15 bytes either side of [src, src+len) inside the same 16-byte granules,
// which is always inside the caller's allocation (cudaMalloc granularity >= 256 B).
__device__ __forceinline__ uint32_t zb_stage_chunk(uint8_t *buf, const uint8_t *src, uint32_t len,
                                                   uint64_t *bar) {
  uint32_t mis = (uint32_t)((uintptr_t)src & 15u);
  uint32_t bytes = (mis + len + 15u) & ~15u;
  if (bytes == 0) bytes = 16;
  zb_mbar_expect_tx(bar, bytes);
  // a single bulk copy is limited by the mbarrier tx-count width; split into 32 KiB pieces
  const uint8_t *g = src - mis;
  uint32_t done = 0;
  while (done < bytes) {
    uint32_t n = bytes - done;
    if (n > 32768u) n = 32768u;
    zb_tma_load_1d(buf + done, g + done, n, bar);
    done += n;
  }
  return mis;
}

// ---- unaligned little-endian reads from shared memory ----
__device__ __forceinline__ uint32_t zb_ld32_unaligned(const uint8_t *base, uint32_t off) {
  const uint32_t *w = reinterpret_cast<const uint32_t *>(base) + (off >> 2);
  uint32_t lo = w[0], hi = w[1];
  return __funnelshift_r(lo, hi, (off & 3u) * 8u);
}

// ---- warp XOR / add reductions ----
__device__ __forceinline__ uint32_t zb_warp_xor(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(ZB_FULL, v, o);
  return v;
}
__device__ __forceinline__ uint64_t zb_warp_sum64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ZB_FULL, v, o);
  return v;
}

// `ts` = distance (in words) between consecutive table entries: 1 for the plain [4][256] table, 32 for the
// per-lane copies the checksum kernel keeps (pass tab + lane there)
__device__ __forceinline__ uint32_t zb_mul1024(const uint32_t *tab /*[4][256] in smem*/, uint32_t r, uint32_t ts = 1u) {
  return tab[(r & 255u) * ts] ^ tab[(256 + ((r >> 8) & 255u)) * ts] ^ tab[(512 + ((r >> 16) & 255u)) * ts] ^ tab[(768 + (r >> 24)) * ts];
}

// Raw (init-0) CRC-32 and Adler sums of bytes [off, off+n) of a shared-memory buffer,
// computed by one warp: lane i takes 32-bit words i, i+32, ... of each 128-byte row,
// advances its state by x^1024 per row (4 table lookups), then the lane states are
// shifted by x^(32*(32-i)) and XOR-reduced.  Result is uniform across the warp.
// a_sum = sum of bytes, b_sum = sum (n - i) * b_i  (exact, 64-bit).
struct ZbCheck {
  uint32_t crc_raw;
  uint64_t a_sum, b_sum;
};
// FULL = the piece size with the fast path, QOFF = where its quarter shifts x^(8 * FULL/4 * k), k = 0..3, sit in lane_mul.
// WANT = which sums are computed (ZB_CK_CRC | ZB_CK_ADLER); the other fields of the result are 0.
#define ZB_CK_CRC 1
#define ZB_CK_ADLER 2
template <uint32_t FULL = ZB_SUB_BYTES, int QOFF = 41, int WANT = ZB_CK_CRC | ZB_CK_ADLER>
__device__ __forceinline__ ZbCheck zb_warp_checksums(const uint8_t *base, uint32_t off, uint32_t n,
                                                     const uint32_t *tab, const uint32_t *lane_mul, uint32_t ts = 1u) {
  const int lane = zb_lane();
  if (ts != 1u) tab += lane;
  if (n == FULL && ts == 1u) {
    // Full piece (the common case): four independent Horner chains of FULL/512 rows each, so the
    // table-lookup latency of one chain hides behind the other three; they are joined with the
    // quarter shifts lane_mul[QOFF + k] = x^(8 * FULL/4 * k).
    uint32_t r0 = 0, r1 = 0, r2 = 0, r3 = 0, a = 0;
    uint64_t b = 0;
    const uint32_t o = off + 4u * (uint32_t)lane, rel0 = 4u * (uint32_t)lane;
    constexpr uint32_t QR = FULL / 512;  // rows of 128 B per quarter
    constexpr uint32_t QB = FULL / 4;    // bytes per quarter
#pragma unroll 2
    for (uint32_t k = 0; k < QR; k++) {
      const uint32_t w0 = zb_ld32_unaligned(base, o + 128u * k), w1 = zb_ld32_unaligned(base, o + 128u * (QR + k));
      const uint32_t w2 = zb_ld32_unaligned(base, o + 128u * (2u * QR + k)), w3 = zb_ld32_unaligned(base, o + 128u * (3u * QR + k));
      if (WANT & ZB_CK_CRC) {
        if (k) {
          r0 = zb_mul1024(tab, r0);
          r1 = zb_mul1024(tab, r1);
          r2 = zb_mul1024(tab, r2);
          r3 = zb_mul1024(tab, r3);
        }
        r0 ^= w0;
        r1 ^= w1;
        r2 ^= w2;
        r3 ^= w3;
      }
      if (!(WANT & ZB_CK_ADLER)) continue;
      const uint32_t s0 = __dp4a(w0, 0x01010101u, 0u), s1 = __dp4a(w1, 0x01010101u, 0u);
      const uint32_t s2 = __dp4a(w2, 0x01010101u, 0u), s3 = __dp4a(w3, 0x01010101u, 0u);
      a += s0 + s1 + s2 + s3;
      const uint32_t rel = rel0 + 128u * k;
      b += (uint64_t)(4u * QB - rel) * s0 + (uint64_t)(3u * QB - rel) * s1 + (uint64_t)(2u * QB - rel) * s2 +
           (uint64_t)(QB - rel) * s3;
      b -= (uint64_t)(__dp4a(w0, 0x03020100u, 0u) + __dp4a(w1, 0x03020100u, 0u) + __dp4a(w2, 0x03020100u, 0u) +
                      __dp4a(w3, 0x03020100u, 0u));
    }
    ZbCheck out;
    out.crc_raw = 0;
    out.a_sum = out.b_sum = 0;
    if (WANT & ZB_CK_CRC) {
      uint32_t r = zb_gf2_mul(r0, lane_mul[QOFF + 3]) ^ zb_gf2_mul(r1, lane_mul[QOFF + 2]) ^ zb_gf2_mul(r2, lane_mul[QOFF + 1]) ^ r3;
      r = zb_gf2_mul(r, lane_mul[32 - lane]);
      out.crc_raw = zb_warp_xor(r);
    }
    if (WANT & ZB_CK_ADLER) {
      out.a_sum = zb_warp_sum64((uint64_t)a);
      out.b_sum = zb_warp_sum64(b);
    }
    return out;
  }
  const uint32_t rows = n >> 7, tail = n & 127u;
  uint32_t r = 0;
  uint32_t a = 0;
  uint64_t b = 0;
  uint32_t o = off + 4u * (uint32_t)lane;  // byte offset of this lane's word in row 0
  uint32_t rel = 4u * (uint32_t)lane;      // offset relative to the piece start
  for (uint32_t k = 0; k < rows; k++) {
    uint32_t w = zb_ld32_unaligned(base, o);
    if (k) r = zb_mul1024(tab, r, ts);
    r ^= w;
    uint32_t s = __dp4a(w, 0x01010101u, 0u);
    uint32_t ws = __dp4a(w, 0x03020100u, 0u);
    a += s;
    b += (uint64_t)(n - rel) * s - ws;
    o += 128u;
    rel += 128u;
  }
  uint32_t crc = rows ? zb_gf2_mul(r, lane_mul[32 - lane]) : 0u;
  // tail: < 128 bytes = tw full words (one per lane) + rem bytes (lane 0, bitwise)
  const uint32_t tw = tail >> 2, rem = tail & 3u;
  uint32_t crc_tail = 0;
  if ((uint32_t)lane < tw) {
    uint32_t w = zb_ld32_unaligned(base, o);
    crc_tail = zb_gf2_mul(w, lane_mul[tw - (uint32_t)lane]);
    uint32_t s = __dp4a(w, 0x01010101u, 0u);
    uint32_t ws = __dp4a(w, 0x03020100u, 0u);
    a += s;
    b += (uint64_t)(n - rel) * s - ws;
  }
  uint32_t crc_rem = 0;
  if (lane == 0) {
    for (uint32_t i = 0; i < rem; i++) {
      uint32_t byte = base[off + (rows << 7) + 4u * tw + i];
      crc_rem = zb_crc_raw_byte(crc_rem, byte);
      a += byte;
      b += (uint64_t)(rem - i) * byte;
    }
  }
  ZbCheck out;
  out.crc_raw = 0;
  out.a_sum = out.b_sum = 0;
  if (WANT & ZB_CK_CRC) {
    crc = zb_warp_xor(crc);
    crc_tail = zb_warp_xor(crc_tail);
    crc_rem = __shfl_sync(ZB_FULL, crc_rem, 0);
    uint32_t raw = crc;
    if (tail) {
      raw = zb_gf2_mul(crc, zb_xpow8(tail));
      if (rem) raw ^= zb_gf2_mul(crc_tail, zb_xpow8(rem)) ^ crc_rem;
      else raw ^= crc_tail;
    }
    out.crc_raw = raw;
  }
  if (WANT & ZB_CK_ADLER) {
    out.a_sum = zb_warp_sum64((uint64_t)a);
    out.b_sum = zb_warp_sum64(b);
  }
  return out;
}
