/* lz2_filtered_model.c -- lz2_model.c's parse with a minimum match length: ZB200_STRATEGY_FILTERED runs k_lz2 with
 * minimum 6 (zlib deflate_slow's match_length <= 5 rule).  A lane's longest candidate shorter than the minimum counts
 * as no match before the one-step lazy rule compares neighbouring lanes; every other rule, constant and the token
 * encoding are lz2_model.c's, which this file includes.  filtered_chunk is model_chunk with that one added line. */
#include "lz2_model.c"

static void filtered_chunk(State *S, const Params *P, uint32_t minm) {
  const uint8_t *R = S->R;
  const uint32_t hb = S->hb, len = S->len, rlen = hb + len;
  static uint16_t stat[NSEG_MAX][1 << STATIC_BITS];
  static uint16_t own[1 << OWN_BITS][WAYS];

  /* static tables: every region segment but the last; entry = the highest q of the segment with that hash */
  const uint32_t nseg = (rlen + SUB - 1) / SUB;
  for (uint32_t sg = 0; sg + 1 < nseg; sg++) {
    memset(stat[sg], 0xff, sizeof stat[sg]);
    for (uint32_t q = sg * SUB; q < (sg + 1) * SUB; q++)
      if (q + 4 <= rlen) stat[sg][hash_static(rd32(R + q))] = (uint16_t)q;
  }

  for (uint32_t b0 = 0; b0 < len; b0 += SUB) {
    const uint32_t b1 = b0 + SUB < len ? b0 + SUB : len;
    const uint32_t myseg = (hb + b0) / SUB;
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
          for (int j = 0; j < P->hist_segs; j++) {
            ce[nc] = myseg > (uint32_t)j ? stat[myseg - 1 - j][hs[l]] : 0xffffu;
            ck[nc++] = K_STATIC;
          }
          /* verify: distance in range, four bytes equal; at most LIST survivors */
          uint32_t dl[LIST];
          int dk[LIST], nl = 0;
          const uint32_t maxd = q < MAXD ? q : MAXD;
          for (int i = 0; i < nc; i++) {
            const uint32_t d = (q - ce[i]) & 0xffffu;
            if (d - 1u >= maxd) continue;
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
          if (m[l] < minm) m[l] = 0;  /* the only rule that differs from model_chunk */
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

/* lz2_model with minimum match length min_len (4: exactly lz2_model's tokens). */
EXPORT int64_t lz2_model_min(const uint8_t *member, uint64_t n, int level, uint32_t *tok, uint64_t cap,
                             uint32_t *chunk_ntok, uint64_t *counters, int min_len) {
  const Params *P = &PARAMS[(level >= 2 && level <= 9) ? level : 6];
  State S;
  memset(&S, 0, sizeof S);
  S.member = member;
  S.n = n;
  S.tok = tok;
  S.cap = cap;
  S.cnt = counters;
  uint64_t nchunks = n == 0 ? 1 : (n + CHUNK - 1) / CHUNK;
  for (uint64_t k = 0; k < nchunks; k++) {
    const uint64_t before = S.ntok;
    S.c0 = k * CHUNK;
    S.hb = (uint32_t)(S.c0 < HIST ? S.c0 : HIST);
    S.len = (uint32_t)(n - S.c0 < CHUNK ? n - S.c0 : CHUNK);
    S.R = member + S.c0 - S.hb;
    filtered_chunk(&S, P, (uint32_t)min_len);
    chunk_ntok[k] = (uint32_t)(S.ntok - before);
  }
  return S.overflow ? -1 : (int64_t)S.ntok;
}
