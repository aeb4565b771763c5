// rsync_model.c -- a sequential CPU model of the rsyncable chunk rule (DESIGN.md section 5 "Rsyncable",
// include/zippy_b200.h "rsyncable compression").  It shares no code with the kernel (zippy_b200/csrc/zb_rsync.cu):
// one pass over the member rolls the gear hash, tests each position, keeps the last candidate for the accept test
// and places the starts of every gap.  tests/test_rsyncable_model.py checks it against a direct Python restatement;
// tests/test_gpu_rsyncable.py checks the kernel against it.
#include <stdint.h>

#define EXPORT extern "C"

static const uint64_t kMin = 16384, kChunk = 65536;
static const int kBits = 16;

// G[b]: the (b + 1)-th output of splitmix64 from state 0, generated one step after the other
EXPORT void rs_model_gear(uint64_t *g) {
  uint64_t state = 0;
  for (int b = 0; b < 256; b++) {
    state += 0x9E3779B97F4A7C15ull;
    uint64_t z = state;
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    g[b] = z;
  }
}

// every candidate p (0 < p < len, h(p) >> 48 == 0), ascending; returns their number (only the first cap are stored)
EXPORT uint64_t rs_model_candidates(const uint8_t *m, uint64_t len, uint64_t *out, uint64_t cap) {
  uint64_t g[256];
  rs_model_gear(g);
  uint64_t h = 0, n = 0;
  for (uint64_t p = 0; p < len; p++) {
    if (p > 0 && (h >> (64 - kBits)) == 0) {
      if (n < cap) out[n] = p;
      n++;
    }
    h = (h << 1) + g[m[p]];
  }
  return n;
}

// the member's chunk starts, ascending from 0; returns their number (only the first cap are stored)
EXPORT uint64_t rs_model_chunks(const uint8_t *m, uint64_t len, uint64_t *out, uint64_t cap) {
  uint64_t g[256];
  rs_model_gear(g);
  uint64_t h = 0, n = 0, cut = 0;
  bool have_prev = false;
  uint64_t prev = 0;   // the last candidate so far
  auto gap = [&](uint64_t a, uint64_t b) {
    for (uint64_t s = a; s < b; s += kChunk) {
      if (n < cap) out[n] = s;
      n++;
    }
  };
  for (uint64_t p = 0; p < len; p++) {
    if (p > 0 && (h >> (64 - kBits)) == 0) {
      if (p >= kMin && (!have_prev || p - prev >= kMin)) {
        gap(cut, p);
        cut = p;
      }
      have_prev = true;
      prev = p;
    }
    h = (h << 1) + g[m[p]];
  }
  if (len == 0) gap(0, 1);
  else gap(cut, len);
  return n;
}
