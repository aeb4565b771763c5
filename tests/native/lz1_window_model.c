/* lz1_window_model.c -- lz1_model.c's level-1 parse under a window of max_dist bytes (zlib's windowBits: max_dist =
 * 2^n).  It includes lz1_model.c for every shared rule, constant, table and counter, and exports lz1_model too;
 * window_chunk is lz1_model.c's model_chunk for mode 1 with the one rule a window changes: lane p has a match only if
 * p - c <= max_dist (32768 in lz1_model).  Every match of level 1 lies within a 4 KiB piece and its 2 KiB pre-seed,
 * so max_dist >= 6144 gives lz1_model's tokens. */
#include "lz1_model.c"

static void window_chunk(const uint8_t *B, uint32_t len, uint32_t flags, uint32_t maxd, Out *o, uint64_t *edge) {
  uint64_t *cnt = o->cnt;
  const uint32_t minm = (flags & F_LIMIT3) ? 3 : MINM;
  const int links = (flags & F_TWO_ROUNDS) ? 4 : 8;
  static Table T;
  for (uint32_t b0 = 0; b0 < len; b0 += PIECE) {
    const uint32_t b1 = b0 + PIECE < len ? b0 + PIECE : len;
    const uint32_t sbase = b0 >= PHASE ? PHASE - PHASE_HIST : 0;
    uint32_t pre = b0 - sbase < PRESEED ? b0 - sbase : PRESEED;
    if (flags & F_PRESEED_2K) pre = b0 < PRESEED ? b0 : PRESEED;
    uint32_t entry = b0;
    memset(T.pos, 0xff, sizeof T.pos);
    memset(T.contested, 0, sizeof T.contested);
    for (uint32_t s = b0 - pre; s < b0; s += 32) {
      uint32_t h[32];
      int ok[32];
      for (int l = 0; l < 32; l++) {
        const uint32_t p = s + (uint32_t)l;
        ok[l] = p + 4 <= len;
        h[l] = ok[l] ? lz_hash(rd32(B + p)) : 0;
      }
      store32(&T, s, h, ok, (flags & F_LOWEST) != 0, cnt);
    }
    for (uint32_t wb = b0; wb < b1; wb += 32) {
      cnt[C_WINDOWS]++;
      if (entry >= wb + 32) {
        cnt[C_SKIPPED]++;
        continue;
      }
      cnt[C_ENTERED]++;
      const uint32_t nvalid = b1 - wb < 32 ? b1 - wb : 32;
      const uint32_t cur = entry - wb;
      uint32_t m[32], dist[32];
      memset(m, 0, sizeof m);
      {
        uint32_t h[32], c[32], steps_max = 0;
        int ok[32];
        for (int l = 0; l < 32; l++) {   /* every lane probes ... */
          const uint32_t p = wb + (uint32_t)l;
          ok[l] = p + 4 <= len;
          h[l] = ok[l] ? lz_hash(rd32(B + p)) : 0;
          c[l] = T.pos[h[l]];
        }
        for (int l = 0; l < 32; l++) {
          const uint32_t p = wb + (uint32_t)l;
          const uint32_t limit = p < b1 ? (b1 - p < MAXM ? b1 - p : MAXM) : 0;
          if (!(ok[l] && p >= entry && limit >= minm)) continue;
          if (T.contested[h[l]]) cnt[C_CONTESTED_READS]++;
          if (!(c[l] < p && p - c[l] <= maxd)) continue;   /* the window */
          if (memcmp(B + c[l], B + p, 4) != 0) {
            cnt[C_COLLISIONS]++;
            continue;
          }
          cnt[C_VERIFIED]++;
          const uint32_t m32 = prefix(B + c[l], B + p, len - p < CAP ? len - p : CAP);
          const uint32_t steps = m32 >= CAP ? CAP / 4 - 1 : m32 / 4;
          cnt[C_EXT_STEPS_LANES] += steps;
          if (steps > steps_max) steps_max = steps;
          m[l] = m32 < CAP ? (m32 < limit ? m32 : limit) : m32;
          dist[l] = p - c[l];
        }
        cnt[C_EXT_STEPS_WARP] += steps_max;
        store32(&T, wb, h, ok, (flags & F_LOWEST) != 0, cnt);   /* ... then every lane stores */
      }
      /* the greedy chain from cur */
      int sel[8], nsel = 0;
      for (uint32_t l = cur; l < 32 && nsel < links;) {
        if (!m[l]) {
          l++;
          continue;
        }
        sel[nsel++] = (int)l;
        l += m[l];
      }
      uint32_t pos = cur, endw = 0;
      for (int i = 0; i < nsel; i++) {
        const uint32_t l = (uint32_t)sel[i], p = wb + l, d = dist[l];
        uint32_t mlen = m[l];
        if (i == nsel - 1 && mlen >= CAP) {
          const uint32_t lim = b1 - p < MAXM ? b1 - p : MAXM;
          mlen = (flags & F_NO_EXIT_EXT) ? (lim < CAP ? lim : CAP) : prefix(B + p - d, B + p, lim);
          cnt[C_CAP_EXT]++;
        }
        for (; pos < l; pos++) emit(o, B[wb + pos]);
        cnt[C_MATCHES]++;
        if (d == maxd) (*edge)++;
        if (p - d < b0) cnt[C_PRESEED_HITS]++;
        if (p - d < b0 && b0 == PHASE) cnt[C_PRESEED_SHORT]++;
        if (mlen == MAXM) cnt[C_M258]++;
        if (p + mlen == b1 && b1 < len && mlen < MAXM && B[b1] == B[b1 - d]) cnt[C_LIMIT_CUT]++;
        emit(o, mlen << 16 | d);
        pos = l + mlen;
        endw = pos;
      }
      if (nsel == 8) cnt[C_WIN8]++;
      for (; pos < nvalid; pos++) emit(o, B[wb + pos]);
      entry = wb + (endw > nvalid ? endw : nvalid);
    }
  }
}

/* lz1_model(member, n, 1, flags, ...) with matches at most max_dist back; *edge receives the number of selected
 * matches at exactly max_dist.  Tokens, chunk_ntok, counters and the return value as for lz1_model. */
EXPORT int64_t lz1_window_model(const uint8_t *member, uint64_t n, uint32_t flags, uint32_t max_dist, uint32_t *tok,
                                uint64_t cap, uint32_t *chunk_ntok, uint64_t *counters, uint64_t *edge) {
  Out o;
  memset(&o, 0, sizeof o);
  o.tok = tok;
  o.cap = cap;
  o.cnt = counters;
  *edge = 0;
  const uint64_t nchunks = n == 0 ? 1 : (n + CHUNK - 1) / CHUNK;
  for (uint64_t k = 0; k < nchunks; k++) {
    const uint64_t before = o.ntok, c0 = k * CHUNK;
    window_chunk(member + c0, (uint32_t)(n - c0 < CHUNK ? n - c0 : CHUNK), flags, max_dist, &o, edge);
    chunk_ntok[k] = (uint32_t)(o.ntok - before);
  }
  return o.overflow ? -1 : (int64_t)o.ntok;
}
