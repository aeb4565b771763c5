/* lz2_model.c -- a sequential CPU model of the parse that k_lz2 makes for levels -1 (Default) and 2..9.
 *
 * An independent restatement of the rules in DESIGN.md sections 4 and 5; it includes nothing from the kernel.
 * It processes one member, chunk by chunk, one 8 KiB sub-chunk and one 32-position window at a time, and
 * writes the tokens each chunk's DEFLATE block must hold:
 *   a literal byte b   -> b                  (< 256)
 *   a match            -> length << 16 | distance  (length 4..258, distance 1..32768)
 *
 * Chunk k covers member bytes [65536 k, 65536 k + len) and sees hb = min(32768, 65536 k) bytes of history in
 * front; region position q = hb + p for chunk position p.  Every rule reads only region bytes before the end
 * of the position's sub-chunk, so the tokens are a function of the member alone.
 *
 * Counters (what the member exercised, summed over its chunks) are reported so a test can show that a
 * comparison reached every rule. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef __cplusplus
#define EXPORT extern "C"
#else
#define EXPORT
#endif

enum { CHUNK = 65536, SUB = 8192, HIST = 32768, MAXM = 258, MINM = 4, MAXD = 32768, CAP = 32, LIST = 8, WAYS = 4 };
enum { OWN_BITS = 11, STATIC_BITS = 13, NSEG_MAX = (CHUNK + HIST) / SUB };
enum { K_WINDOW = 0, K_OWN = 1, K_STATIC = 2 };

/* counter slots */
enum {
  C_MATCHES,      /* selected matches */
  C_LAZY_DROPS,   /* matches dropped by the one-step lazy rule */
  C_HISTORY,      /* selected matches whose source lies before the chunk */
  C_DIST_32768,   /* selected matches at distance 32768 */
  C_CAP_EXT,      /* last matches of a window that reached the lane cap and were extended */
  C_LIMIT_CUT,    /* selected matches that end at the sub-chunk end although the bytes go on matching */
  C_SHORT_LIMIT,  /* selected matches whose limit was 4..31 */
  C_WIN_WINDOW,   /* selected matches found through the nearest same-hash position of the window */
  C_WIN_OWN,      /* ... through the sub-chunk's own table */
  C_WIN_STATIC,   /* ... through a preceding segment's static table */
  C_ALIAS,        /* empty table entries (0xffff) that passed the distance test and were compared */
  C_258_AT_END,   /* selected 258-byte matches that end exactly at the sub-chunk end */
  C_COUNT
};

typedef struct {
  int own_ways, hist_segs, maxcand, good, lazy;
} Params;

/* own hist maxcand good lazy, by level; -1 (Default) is level 6 */
static const Params PARAMS[10] = {{4, 4, 4, 8, 16}, {4, 4, 4, 8, 16}, {2, 4, 2, 4, 0},  {2, 4, 3, 4, 6},  {3, 4, 3, 4, 8},
                                  {3, 4, 4, 8, 16}, {4, 4, 4, 8, 16}, {4, 4, 6, 8, 32}, {4, 4, 8, 16, 32}, {4, 4, 8, 32, 64}};

static uint32_t rd32(const uint8_t *b) { return (uint32_t)b[0] | (uint32_t)b[1] << 8 | (uint32_t)b[2] << 16 | (uint32_t)b[3] << 24; }
static uint32_t hash_own(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - OWN_BITS); }
static uint32_t hash_static(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - STATIC_BITS); }

/* common prefix of a[0..] and b[0..], at most n */
static uint32_t prefix(const uint8_t *a, const uint8_t *b, uint32_t n) {
  uint32_t k = 0;
  while (k < n && a[k] == b[k]) k++;
  return k;
}

typedef struct {
  const uint8_t *member;
  uint64_t n, c0;            /* member length, chunk start in the member */
  const uint8_t *R;          /* region: R[q] = member[c0 - hb + q] */
  uint32_t hb, len;
  uint32_t *tok;
  uint64_t ntok, cap;
  uint64_t *cnt;
  int overflow;
} State;

static void emit(State *S, uint32_t t) {
  if (S->ntok < S->cap) S->tok[S->ntok] = t;
  else S->overflow = 1;
  S->ntok++;
}

static void emit_match(State *S, uint32_t p, uint32_t len, uint32_t d, uint32_t b1, int kind, int extended,
                       uint32_t limit) {
  uint64_t *c = S->cnt;
  c[C_MATCHES]++;
  if (d > p) c[C_HISTORY]++;
  if (d == MAXD) c[C_DIST_32768]++;
  if (extended) c[C_CAP_EXT]++;
  if (limit < CAP) c[C_SHORT_LIMIT]++;
  if (len == b1 - p && len < MAXM) {
    const uint64_t at = S->c0 + p + len;  /* the byte after the match, in the member */
    if (at < S->n && S->member[at] == S->member[at - d]) c[C_LIMIT_CUT]++;
  }
  if (len == MAXM && p + MAXM == b1) c[C_258_AT_END]++;
  c[kind == K_WINDOW ? C_WIN_WINDOW : kind == K_OWN ? C_WIN_OWN : C_WIN_STATIC]++;
  emit(S, len << 16 | d);
}

static void model_chunk(State *S, const Params *P) {
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

/* Parse one member at `level`.  chunk_ntok[k] receives the number of tokens of chunk k (room for
 * max(1, ceil(n / 65536)) entries); counters has C_COUNT slots and is added to.  Returns the total number
 * of tokens, or -1 when `cap` is too small (nothing beyond cap is written). */
EXPORT int64_t lz2_model(const uint8_t *member, uint64_t n, int level, uint32_t *tok, uint64_t cap,
                         uint32_t *chunk_ntok, uint64_t *counters) {
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
    model_chunk(&S, P);
    chunk_ntok[k] = (uint32_t)(S.ntok - before);
  }
  return S.overflow ? -1 : (int64_t)S.ntok;
}

EXPORT int lz2_counter_count(void) { return C_COUNT; }
