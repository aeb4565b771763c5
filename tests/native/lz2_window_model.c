/* lz2_window_model.c -- the parse of k_lz2 (lz2_model.c) under a window of max_dist bytes (zlib's windowBits:
 * max_dist = 2^n), for members (lz2_model), the FILTERED minimum length (lz2_filtered_model.c) and a flushed stream's
 * chunk schedule (lz2_schedule_model.c) alike.
 *
 * It includes lz2_model.c for every shared rule, constant, hash, counter and the token emission, and exports lz2_model
 * too.  window_chunk is lz2_schedule_model.c's model_chunk_grid (for a history that is a multiple of SUB, hg = 0 and it
 * is lz2_model.c's model_chunk) with the minimum match length of lz2_filtered_model.c and the two rules a window
 * changes:
 *   - a candidate is in range at distance 1..min(q, max_dist) (32768 in lz2_model);
 *   - a preceding segment j (0 = nearest) holds only positions more than SUB * j back, so its static table is looked
 *     up only when SUB * j < max_dist: hist_segs is at most ceil(max_dist / SUB).  A slot not looked up is not a
 *     candidate at all (an empty entry would alias to distance (q + 1) mod 2^16, which can lie in range).
 * At max_dist 32768 and minimum 4 the tokens are lz2_model's (and lz2_model_schedule's for a schedule). */
#include "lz2_model.c"

static void window_chunk(State *S, const Params *P, uint32_t minm, uint32_t maxd, uint64_t *edge) {
  const uint8_t *R = S->R;
  const uint32_t hb = S->hb, len = S->len, rlen = hb + len;
  const uint32_t hg = (SUB - hb % SUB) % SUB;
  const int segs = (int)((maxd + SUB - 1) / SUB), hist_segs = P->hist_segs < segs ? P->hist_segs : segs;
  static uint16_t stat[NSEG_MAX][1 << STATIC_BITS];
  static uint16_t own[1 << OWN_BITS][WAYS];

  /* static tables: every segment of the grid but the last; entry = the highest q of the segment with that hash */
  const uint32_t nseg = (hg + rlen + SUB - 1) / SUB;
  for (uint32_t sg = 0; sg + 1 < nseg; sg++) {
    memset(stat[sg], 0xff, sizeof stat[sg]);
    for (uint32_t q = sg ? sg * SUB - hg : 0; q < (sg + 1) * SUB - hg; q++)
      if (q + 4 <= rlen) stat[sg][hash_static(rd32(R + q))] = (uint16_t)q;
  }

  for (uint32_t b0 = 0; b0 < len; b0 += SUB) {
    const uint32_t b1 = b0 + SUB < len ? b0 + SUB : len;
    const uint32_t myseg = (hg + hb + b0) / SUB;
    memset(own, 0xff, sizeof own);
    uint32_t entry = b0;
    for (uint32_t wb = b0; wb < b1; wb += 32) {
      int can[32];
      uint32_t h[32], hs[32], bucket[32][WAYS];
      for (int l = 0; l < 32; l++) {
        const uint32_t p = wb + (uint32_t)l;
        can[l] = p + 4 <= len;
        if (!can[l]) continue;
        const uint32_t v = rd32(R + hb + p);
        h[l] = hash_own(v);
        hs[l] = hash_static(v);
        for (int w = 0; w < WAYS; w++) bucket[l][w] = own[h[l]][w];  /* as it was before this window */
      }
      if (entry < wb + 32) {
        const uint32_t nvalid = b1 - wb < 32 ? b1 - wb : 32;
        const uint32_t cur = entry - wb;
        uint32_t m[32], dist[32], lim[32];
        int kind[32];
        for (int l = 0; l < 32; l++) {
          const uint32_t p = wb + (uint32_t)l, q = hb + p;
          m[l] = 0;
          dist[l] = 1;
          kind[l] = K_WINDOW;
          lim[l] = p < b1 ? (b1 - p < MAXM ? b1 - p : MAXM) : 0;
          if (!(can[l] && p >= entry && lim[l] >= MINM)) continue;
          /* candidates, in order */
          uint32_t ce[1 + WAYS + 4];
          int ck[1 + WAYS + 4], nc = 0;
          for (int j = l - 1; j >= 0; j--)
            if (can[j] && h[j] == h[l]) {
              ce[nc] = q - (uint32_t)(l - j);
              ck[nc++] = K_WINDOW;
              break;
            }
          for (int w = 0; w < P->own_ways; w++) {
            ce[nc] = bucket[l][w];
            ck[nc++] = K_OWN;
          }
          for (int j = 0; j < hist_segs; j++) {
            ce[nc] = myseg > (uint32_t)j ? stat[myseg - 1 - j][hs[l]] : 0xffffu;
            ck[nc++] = K_STATIC;
          }
          /* verify: distance in range, four bytes equal; at most LIST survivors */
          uint32_t dl[LIST];
          int dk[LIST], nl = 0;
          const uint32_t maxq = q < maxd ? q : maxd;
          for (int i = 0; i < nc; i++) {
            const uint32_t d = (q - ce[i]) & 0xffffu;
            if (d - 1u >= maxq) continue;
            if (ce[i] == 0xffffu && ck[i] != K_WINDOW) S->cnt[C_ALIAS]++;
            if (memcmp(R + q - d, R + q, 4) != 0) continue;
            if (nl < LIST) {
              dl[nl] = d;
              dk[nl++] = ck[i];
            }
          }
          /* extend, nearest first, under the level's budget; lengths clamped to min(limit, lane cap) */
          const uint32_t stop = lim[l] < CAP ? lim[l] : CAP;
          int budget = P->maxcand;
          for (int i = 0; i < nl && budget > 0 && m[l] < stop; i++) {
            const uint32_t d = dl[i];
            budget--;
            if (m[l] >= 4 && R[q - d + m[l]] != R[q + m[l]]) {
              if (m[l] >= (uint32_t)P->good && budget > 1) budget = 1;
              continue;
            }
            const uint32_t mc = prefix(R + q - d, R + q, stop);
            if (mc > m[l]) {
              m[l] = mc;
              dist[l] = d;
              kind[l] = dk[i];
            }
            if (m[l] >= (uint32_t)P->good && budget > 1) budget = 1;
          }
          if (m[l] < minm) m[l] = 0;
        }
        /* one-step lazy evaluation, on the values from before this step */
        uint32_t mz[32];
        for (int l = 0; l < 32; l++) {
          mz[l] = m[l];
          if (l < 31 && m[l] != 0 && m[l] < (uint32_t)P->lazy && m[l + 1] > m[l]) {
            mz[l] = 0;
            S->cnt[C_LAZY_DROPS]++;
          }
        }
        /* greedy selection from the entry; the last match of the window finishes past the lane cap */
        uint32_t pos = cur, endw = 0;
        int l = (int)cur;
        while (l < 32) {
          while (l < 32 && mz[l] == 0) l++;
          if (l == 32) break;
          const uint32_t p = wb + (uint32_t)l;
          uint32_t mlen = mz[l];
          int extended = 0;
          if (mlen >= CAP) {
            mlen = prefix(R + hb + p - dist[l], R + hb + p, lim[l]);
            extended = 1;
          }
          for (; pos < (uint32_t)l; pos++) emit(S, R[hb + wb + pos]);
          emit_match(S, p, mlen, dist[l], b1, kind[l], extended, lim[l]);
          if (dist[l] == maxd) (*edge)++;
          pos = (uint32_t)l + mlen;
          endw = pos;
          l = (int)pos;
        }
        for (; pos < nvalid; pos++) emit(S, R[hb + wb + pos]);
        entry = wb + (endw > nvalid ? endw : nvalid);
      }
      /* every window inserts its positions, in order, whether or not it was parsed */
      for (int l = 0; l < 32; l++) {
        if (!can[l]) continue;
        uint16_t *b = own[h[l]];
        memmove(b + 1, b, (WAYS - 1) * sizeof *b);
        b[0] = (uint16_t)(hb + wb + (uint32_t)l);
      }
    }
  }
}

/* Parse one member at `level` with minimum match length min_len (4; FILTERED: 6) and matches at most max_dist back,
 * under an explicit chunk schedule as lz2_model_schedule takes it (bounds / hist_from, nchunks entries), or with
 * bounds null under lz2_model's (64 KiB chunks, hb = min(32768, chunk start)).  *edge receives the number of selected
 * matches at exactly max_dist.  Tokens, chunk_ntok, counters and the return value as for lz2_model; -2 for a
 * malformed schedule. */
EXPORT int64_t lz2_window_model(const uint8_t *member, uint64_t n, int level, int min_len, uint32_t max_dist,
                                const uint64_t *bounds, const uint64_t *hist_from, uint64_t nchunks, uint32_t *tok,
                                uint64_t cap, uint32_t *chunk_ntok, uint64_t *counters, uint64_t *edge) {
  const Params *P = &PARAMS[(level >= 2 && level <= 9) ? level : 6];
  if (!bounds) nchunks = n == 0 ? 1 : (n + CHUNK - 1) / CHUNK;
  if (bounds) {
    if (nchunks == 0 || bounds[0] != 0 || bounds[nchunks] != n) return -2;
    for (uint64_t k = 0; k < nchunks; k++) {
      const uint64_t len = bounds[k + 1] - bounds[k];
      if (bounds[k + 1] < bounds[k] || len > CHUNK || (len == 0 && k + 1 != nchunks) || hist_from[k] > bounds[k])
        return -2;
    }
  }
  State S;
  memset(&S, 0, sizeof S);
  S.member = member;
  S.n = n;
  S.tok = tok;
  S.cap = cap;
  S.cnt = counters;
  *edge = 0;
  for (uint64_t k = 0; k < nchunks; k++) {
    const uint64_t before = S.ntok;
    S.c0 = bounds ? bounds[k] : k * CHUNK;
    const uint64_t h = bounds ? bounds[k] - hist_from[k] : S.c0;
    S.hb = (uint32_t)(h < HIST ? h : HIST);
    S.len = (uint32_t)(bounds ? bounds[k + 1] - bounds[k] : (n - S.c0 < CHUNK ? n - S.c0 : CHUNK));
    S.R = member + S.c0 - S.hb;
    window_chunk(&S, P, (uint32_t)min_len, max_dist, edge);
    chunk_ntok[k] = (uint32_t)(S.ntok - before);
  }
  return S.overflow ? -1 : (int64_t)S.ntok;
}
