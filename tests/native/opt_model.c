/* opt_model.c -- a sequential CPU model of the optimal parse (k_opt, zb200_compress_batch_optimal).
 *
 * A restatement of the rules in DESIGN.md sections 4 and 5.  The only thing it shares with the library is the
 * code-length builder (zb_huff_lengths in zb_huff.h): each cost round prices symbols with the lengths that builder
 * gives, and tests/test_host_units.py pins that builder on its own.  Tokens are written per chunk:
 *   a literal byte b   -> b                  (< 256)
 *   a match            -> length << 16 | distance  (length 4..258, distance 1..2^window_bits)
 *
 * The rules, per chunk of up to 64 KiB with hb bytes of history in front (region R = history + chunk; region
 * position q = hb + chunk position p):
 *  - chains: every region position q with q + 4 <= |R| is hashed, h = (le32(R[q..q+3]) * 0x9E3779B1) >> 18, and
 *    linked to the previous region position with the same h when that one is at most 2^window_bits back;
 *  - candidates of p (in its 8 KiB sub-chunk [b0, b1), limit = min(258, b1 - p) >= 4): walk p's chain up to
 *    OPT_WALK links while the distance stays within 2^window_bits; a link whose four bytes equal p's is a hit,
 *    extended to its full length (at most limit); the walk stops after OPT_KEEP hits or a hit of length limit.
 *    A hit is kept when it is longer than every nearer one: the kept hits are the Pareto set, and a length L maps
 *    to the nearest kept hit at least L long;
 *  - costs: integer bits.  A literal costs its symbol's cost, a match (L, d) the cost of L's length symbol plus
 *    its extra bits plus the cost of d's distance symbol plus its extra bits.  Round 1 prices every symbol at its
 *    fixed-code length (RFC 1951 3.2.6: 8 / 9 / 7 / 8 bits, distances 5).  Round r + 1 prices it at the length
 *    zb_huff_lengths gives for round r's histogram of the whole chunk (with one end-of-block, limit 15), and a
 *    symbol that got no code at OPT_UNUSED bits;
 *  - shortest path: per sub-chunk, backwards: cost[b1] = 0, cost[p] = the least of the literal (cost + cost[p+1])
 *    and every match (L, d) of p's candidates (cost + cost[p + L]).  Ties go to the literal, then to the shorter
 *    length (which is also the nearer distance).  The path is walked forwards from b0; no match crosses b1;
 *  - OPT_ROUNDS rounds; the last round's path is the chunk's tokens. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "zb_huff.h"

#ifdef __cplusplus
#define EXPORT extern "C"
#else
#define EXPORT
#endif

enum { CHUNK = 65536, SUB = 8192, HIST = 32768, MAXM = 258, MINM = 4, HBITS = 14 };
enum { OPT_WALK = 16, OPT_KEEP = 8, OPT_ROUNDS = 2, OPT_UNUSED = 13 };

enum {
  C_MATCHES,     /* matches on the final paths */
  C_HISTORY,     /* ... whose source lies before the chunk */
  C_DIST_MAX,    /* ... at distance 2^window_bits */
  C_258_AT_END,  /* ... 258 bytes long, ending at their sub-chunk's end */
  C_TIES,        /* positions of a final round where two choices cost the same */
  C_WALK_CUT,    /* candidate walks cut by OPT_WALK links */
  C_KEEP_CUT,    /* candidate walks stopped by OPT_KEEP hits */
  C_COUNT
};

static uint32_t rd32(const uint8_t *b) { return (uint32_t)b[0] | (uint32_t)b[1] << 8 | (uint32_t)b[2] << 16 | (uint32_t)b[3] << 24; }
static uint32_t hash14(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - HBITS); }
static uint32_t prefix(const uint8_t *a, const uint8_t *b, uint32_t n) {
  uint32_t k = 0;
  while (k < n && a[k] == b[k]) k++;
  return k;
}

typedef struct {
  const uint8_t *R;
  uint32_t hb, len, maxd;
  uint16_t *prevd;   /* [hb + len] */
  uint64_t *cnt;
} Chunk;

static void build_chains(Chunk *C) {
  static int32_t head[1 << HBITS];
  const uint32_t rlen = C->hb + C->len;
  for (int i = 0; i < (1 << HBITS); i++) head[i] = -1;
  for (uint32_t q = 0; q < rlen; q++) {
    C->prevd[q] = 0;
    if (q + 4 > rlen) continue;
    const uint32_t h = hash14(rd32(C->R + q));
    if (head[h] >= 0 && q - (uint32_t)head[h] <= C->maxd) C->prevd[q] = (uint16_t)(q - (uint32_t)head[h]);
    head[h] = (int32_t)q;
  }
}

/* the Pareto set of chunk position p: out[j] = length << 16 | distance, lengths and distances increasing */
static int candidates(const Chunk *C, uint32_t p, uint32_t b1, uint32_t *out, uint64_t *cnt) {
  const uint32_t limit = b1 - p < MAXM ? b1 - p : MAXM;
  if (limit < MINM) return 0;
  const uint8_t *R = C->R;
  const uint32_t q = C->hb + p, v = rd32(R + q);
  uint32_t c = q, best = 0, hits = 0;
  int n = 0, link;
  for (link = 0; link < OPT_WALK; link++) {
    const uint32_t step = C->prevd[c];
    if (step == 0) break;
    c -= step;
    const uint32_t d = q - c;
    if (d > C->maxd) break;
    if (rd32(R + c) != v) continue;
    hits++;
    const uint32_t m = prefix(R + c, R + q, limit);
    if (m > best) {
      best = m;
      out[n++] = m << 16 | d;
    }
    if (hits == OPT_KEEP || best == limit) break;
  }
  if (cnt) {
    if (link == OPT_WALK) cnt[C_WALK_CUT]++;
    else if (hits == OPT_KEEP && best < limit) cnt[C_KEEP_CUT]++;
  }
  return n;
}

static uint32_t dist_code(uint32_t d) {
  const uint32_t v = d - 1;
  if (v < 4) return v;
  int hb = 31 - __builtin_clz(v);
  return 2u * (uint32_t)hb + ((v >> (hb - 1)) & 1u);
}
static uint32_t dist_extra(uint32_t code) { return code < 4 ? 0 : (code >> 1) - 1; }
static uint32_t len_code(uint32_t L) {  /* 0..28 */
  static const uint16_t base[29] = ZB_BASE_LENGTHS;
  int c = 28;
  while (base[c] > L) c--;
  return (uint32_t)c;
}
static uint32_t len_extra(uint32_t code) { return (code < 8 || code == 28) ? 0 : (code >> 2) - 1; }

typedef struct {
  uint32_t ll[ZB_NUM_LITLEN], dd[ZB_NUM_DIST];  /* symbol costs */
  uint32_t lcost[MAXM + 1];                      /* length symbol + extra bits, by length */
  uint32_t dcost_code[ZB_NUM_DIST];              /* distance symbol + extra bits, by code */
} Costs;

static void costs_fixed(Costs *K) {
  for (int s = 0; s < ZB_NUM_LITLEN; s++) K->ll[s] = (uint32_t)zb_fixed_ll_len(s);
  for (int s = 0; s < ZB_NUM_DIST; s++) K->dd[s] = 5;
}
static void costs_from_hist(Costs *K, const uint32_t *llf_in, const uint32_t *df) {
  uint32_t llf[ZB_NUM_LITLEN];
  uint8_t lens[ZB_NUM_LITLEN + ZB_NUM_DIST];
  memcpy(llf, llf_in, sizeof llf);
  llf[256] = 1;
  zb_huff_lengths(llf, ZB_NUM_LITLEN, 15, lens);
  zb_huff_lengths(df, ZB_NUM_DIST, 15, lens + ZB_NUM_LITLEN);
  for (int s = 0; s < ZB_NUM_LITLEN; s++) K->ll[s] = lens[s] ? lens[s] : OPT_UNUSED;
  for (int s = 0; s < ZB_NUM_DIST; s++) K->dd[s] = lens[ZB_NUM_LITLEN + s] ? lens[ZB_NUM_LITLEN + s] : OPT_UNUSED;
}
static void costs_derive(Costs *K) {
  for (uint32_t L = MINM; L <= MAXM; L++) {
    const uint32_t c = len_code(L);
    K->lcost[L] = K->ll[257 + c] + len_extra(c);
  }
  for (uint32_t c = 0; c < ZB_NUM_DIST; c++) K->dcost_code[c] = K->dd[c] + dist_extra(c);
}

typedef struct {
  uint32_t *tok;
  uint64_t ntok, cap;
  int overflow;
} Out;

static void emit(Out *O, uint32_t t) {
  if (O->ntok < O->cap) O->tok[O->ntok] = t;
  else O->overflow = 1;
  O->ntok++;
}

/* One chunk: OPT_ROUNDS rounds; the last one's tokens go to O (when not null); *total receives the last round's
 * path cost summed over the sub-chunks and K_out the costs it priced with. */
static void model_chunk(Chunk *C, Out *O, uint64_t *total, Costs *K_out) {
  const uint32_t len = C->len, hb = C->hb;
  uint32_t *cand = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(len ? len : 1) * OPT_KEEP);
  uint8_t *ncand = (uint8_t *)malloc(len ? len : 1);
  uint32_t *cost = (uint32_t *)malloc(sizeof(uint32_t) * (SUB + 1));
  uint32_t *choice = (uint32_t *)malloc(sizeof(uint32_t) * SUB);  /* length << 16 | distance; length 1: literal */
  build_chains(C);
  for (uint32_t b0 = 0; b0 < len; b0 += SUB) {
    const uint32_t b1 = b0 + SUB < len ? b0 + SUB : len;
    for (uint32_t p = b0; p < b1; p++) ncand[p] = (uint8_t)candidates(C, p, b1, cand + (size_t)p * OPT_KEEP, C->cnt);
  }
  Costs K;
  costs_fixed(&K);
  for (int round = 0; round < OPT_ROUNDS; round++) {
    const int last = round == OPT_ROUNDS - 1;
    costs_derive(&K);
    uint32_t llf[ZB_NUM_LITLEN], df[ZB_NUM_DIST];
    memset(llf, 0, sizeof llf);
    memset(df, 0, sizeof df);
    uint64_t tot = 0;
    for (uint32_t b0 = 0; b0 < len; b0 += SUB) {
      const uint32_t b1 = b0 + SUB < len ? b0 + SUB : len;
      cost[b1 - b0] = 0;
      for (uint32_t p = b1; p-- > b0;) {
        const uint32_t i = p - b0;
        uint32_t best = (K.ll[C->R[hb + p]] + cost[i + 1]) << 9 | 1u, bd = 0;
        int tie = 0;
        uint32_t prevlen = MINM - 1;
        for (int j = 0; j < ncand[p]; j++) {
          const uint32_t e = cand[(size_t)p * OPT_KEEP + j], mlen = e >> 16, d = e & 0xffffu;
          const uint32_t dc = K.dcost_code[dist_code(d)];
          for (uint32_t L = prevlen + 1; L <= mlen; L++) {
            const uint32_t key = (K.lcost[L] + dc + cost[i + L]) << 9 | L;
            if ((key >> 9) == (best >> 9)) tie = 1;
            if (key < best) {
              best = key;
              bd = d;
            }
          }
          prevlen = mlen;
        }
        if (last && tie) C->cnt[C_TIES]++;
        cost[i] = best >> 9;
        choice[i] = (best & 511u) << 16 | bd;
      }
      tot += cost[0];
      for (uint32_t p = b0; p < b1;) {
        const uint32_t ch = choice[p - b0], L = ch >> 16, d = ch & 0xffffu;
        if (L == 1) {
          llf[C->R[hb + p]]++;
          if (last && O) emit(O, C->R[hb + p]);
        } else {
          llf[257 + len_code(L)]++;
          df[dist_code(d)]++;
          if (last) {
            C->cnt[C_MATCHES]++;
            if (d > p) C->cnt[C_HISTORY]++;
            if (d == C->maxd) C->cnt[C_DIST_MAX]++;
            if (L == MAXM && p + L == b1) C->cnt[C_258_AT_END]++;
            if (O) emit(O, L << 16 | d);
          }
        }
        p += L;
      }
    }
    if (last) {
      if (total) *total = tot;
      if (K_out) *K_out = K;
    } else {
      costs_from_hist(&K, llf, df);
    }
  }
  free(cand);
  free(ncand);
  free(cost);
  free(choice);
}

static void chunk_at(Chunk *C, const uint8_t *buf, uint64_t hist0, uint64_t n, int window_bits, uint64_t k,
                     uint16_t *prevd, uint64_t *cnt) {
  const uint64_t c0 = hist0 + k * CHUNK;       /* chunk start in buf */
  const uint64_t before = hist0 + k * CHUNK;   /* bytes in front of it */
  C->hb = (uint32_t)(before < HIST ? before : HIST);
  C->len = (uint32_t)(n - k * CHUNK < CHUNK ? n - k * CHUNK : CHUNK);
  C->R = buf + c0 - C->hb;
  C->maxd = 1u << window_bits;
  C->prevd = prevd;
  C->cnt = cnt;
}

/* Parse n bytes that follow hist0 bytes of history in buf (buf holds hist0 + n bytes): chunk k covers
 * buf[hist0 + 65536 k, ...) and sees min(32768, hist0 + 65536 k) bytes of history.  chunk_ntok receives each
 * chunk's token count (max(1, ceil(n / 65536)) entries); counters (C_COUNT slots) are added to.  Returns the
 * number of tokens, or -1 when cap is too small. */
EXPORT int64_t opt_model(const uint8_t *buf, uint64_t hist0, uint64_t n, int window_bits, uint32_t *tok, uint64_t cap,
                         uint32_t *chunk_ntok, uint64_t *counters) {
  Out O = {tok, 0, cap, 0};
  uint16_t *prevd = (uint16_t *)malloc(sizeof(uint16_t) * (CHUNK + HIST));
  const uint64_t nchunks = n == 0 ? 1 : (n + CHUNK - 1) / CHUNK;
  for (uint64_t k = 0; k < nchunks; k++) {
    const uint64_t before = O.ntok;
    Chunk C;
    chunk_at(&C, buf, hist0, n, window_bits, k, prevd, counters);
    model_chunk(&C, &O, NULL, NULL);
    chunk_ntok[k] = (uint32_t)(O.ntok - before);
  }
  free(prevd);
  return O.overflow ? -1 : (int64_t)O.ntok;
}

/* Chunk k of the same parse: the symbol costs of its last round (ll[286], dd[30]), the candidates of every chunk
 * position (cand[p * OPT_KEEP + j], ncand[p]) and the last round's path cost summed over its sub-chunks. */
EXPORT uint64_t opt_model_chunk(const uint8_t *buf, uint64_t hist0, uint64_t n, int window_bits, uint64_t k,
                                uint32_t *ll, uint32_t *dd, uint32_t *cand, uint8_t *ncand) {
  uint64_t cnt[C_COUNT] = {0}, total = 0;
  uint16_t *prevd = (uint16_t *)malloc(sizeof(uint16_t) * (CHUNK + HIST));
  Chunk C;
  chunk_at(&C, buf, hist0, n, window_bits, k, prevd, cnt);
  Costs K;
  model_chunk(&C, NULL, &total, &K);
  memcpy(ll, K.ll, sizeof K.ll);
  memcpy(dd, K.dd, sizeof K.dd);
  for (uint32_t b0 = 0; b0 < C.len; b0 += SUB) {
    const uint32_t b1 = b0 + SUB < C.len ? b0 + SUB : C.len;
    for (uint32_t p = b0; p < b1; p++) ncand[p] = (uint8_t)candidates(&C, p, b1, cand + (size_t)p * OPT_KEEP, NULL);
  }
  free(prevd);
  return total;
}

/* The bytes the library writes for one chunk holding these tokens (the encoding above): k_huff's choice of the
 * smallest of stored, fixed and dynamic, zb_build_codebook, with each token counted in the sub-chunk it starts in. */
EXPORT uint32_t opt_block_bytes(const uint32_t *tok, uint64_t ntok, uint32_t chunk_len, int is_final) {
  static uint16_t hist[ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS];
  static ZbCodebook cb;
  memset(hist, 0, sizeof hist);
  uint32_t p = 0;
  for (uint64_t i = 0; i < ntok; i++) {
    uint16_t *h = hist + (p / SUB) * ZB_HIST_SYMS;
    if (tok[i] < 256) {
      h[tok[i]]++;
      p++;
    } else {
      h[257 + len_code(tok[i] >> 16)]++;
      h[ZB_NUM_LITLEN + dist_code(tok[i] & 0xffffu)]++;
      p += tok[i] >> 16;
    }
  }
  zb_build_codebook(hist, chunk_len, is_final, -1, &cb);
  return cb.total_bytes;
}

EXPORT int opt_counter_count(void) { return C_COUNT; }
EXPORT int opt_param(int which) { return which == 0 ? OPT_WALK : which == 1 ? OPT_KEEP : which == 2 ? OPT_ROUNDS : OPT_UNUSED; }
