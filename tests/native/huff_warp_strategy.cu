// Test-only entry point to k_huff (zippy_b200/csrc/zb_huff_warp.cuh) with its fixed-only block choice
// (ZB200_STRATEGY_FIXED): tests/test_gpu_strategy.py compares its codebooks with the host builder's force_type 1.
#include "../../zippy_b200/csrc/zb_huff_warp.cuh"

extern "C" {
// hist: n x 8 x 316 u16; lens, finals: n each.  The device codebooks are filled with 0xa5 before the launch.
int t_huff_warp_fixed(const uint16_t *hist, const uint32_t *lens, const int *finals, int n, int level, ZbCodebook *out) {
  ZbChunkDesc *d_desc = nullptr;
  uint16_t *d_hist = nullptr;
  ZbCodebook *d_cb = nullptr;
  ZbChunkDesc *desc = new ZbChunkDesc[n];
  for (int i = 0; i < n; i++) {
    desc[i].src_off = 0;
    desc[i].len = lens[i];
    desc[i].member = (uint32_t)i;
    desc[i].flags = finals[i] ? ZB_CHUNK_LAST : 0u;
    desc[i].pad = 0;
  }
  const size_t hb = (size_t)n * ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS * sizeof(uint16_t);
  cudaError_t e = cudaMalloc(&d_desc, n * sizeof(ZbChunkDesc));
  if (e == cudaSuccess) e = cudaMalloc(&d_hist, hb);
  if (e == cudaSuccess) e = cudaMalloc(&d_cb, n * sizeof(ZbCodebook));
  if (e == cudaSuccess) e = cudaMemcpy(d_desc, desc, n * sizeof(ZbChunkDesc), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_hist, hist, hb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(d_cb, 0xa5, n * sizeof(ZbCodebook));
  if (e == cudaSuccess) {
    k_huff<<<(n + HW_WARPS - 1) / HW_WARPS, HW_WARPS * 32>>>(d_desc, d_hist, d_cb, (uint32_t)n, level, true);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, d_cb, n * sizeof(ZbCodebook), cudaMemcpyDeviceToHost);
  cudaFree(d_desc);
  cudaFree(d_hist);
  cudaFree(d_cb);
  delete[] desc;
  return (int)e;
}
}
