/* lz1_model.c -- a sequential CPU model of the parse that k_lz<1> makes for level 1 (BestSpeed), and of the
 * literals-only parse of k_lz<0> (level -2).
 *
 * An independent restatement of the rules in DESIGN.md section 4; it includes nothing from the kernel.  It
 * processes one member, chunk by chunk, one 4 KiB piece and one 32-position window at a time, and writes the
 * tokens each chunk's DEFLATE block must hold:
 *   a literal byte b   -> b                  (< 256)
 *   a match            -> length << 16 | distance  (length 4..258, distance 1..32768)
 *
 * The rules, for a chunk of len <= 65536 bytes (chunks are independent: a match never reaches before its chunk):
 *   - two phases of 32 KiB, sixteen pieces of 4 KiB; piece [b0, b1) starts with an empty 2048-entry table of u16
 *     positions (0xffff), pre-seeded with [b0 - min(2048, b0 - sbase), b0), where sbase = 0 in phase 0 and
 *     32768 - 1024 in phase 1 (only 1 KiB of phase 0 is staged again).  Hash: (v * 0x9E3779B1) >> 21 of the 4
 *     bytes at p read little-endian.  A position is inserted only if p + 4 <= len.
 *   - windows of 32 positions; a window is entered only if entry < wb + 32 (a skipped window inserts nothing).
 *     In an entered window every lane probes, then every lane with p + 4 <= len stores (also lanes before entry).
 *     Lanes of one store instruction (a window, or 32 positions of the pre-seed) that share an entry: the highest
 *     or the lowest position lands (a parameter: the kernel leaves it to the hardware unless built with
 *     ZB_LZ1_RESOLVE_WINNER=1, which makes the highest win).
 *   - lane p has a match iff c < p, p - c <= 32768, p >= entry, limit = min(258, b1 - p) >= 4 and the 4 bytes at c
 *     and p are equal.  It extends to at most 32 bytes (the lane cap); a length below 32 is clamped to limit.
 *   - greedy chain: the first match at or after cur = entry - wb, then the first match at or after the previous
 *     one's end; three doubling rounds follow at most 8 links.  If the last selected match reached 32 bytes it is
 *     extended to min(258, b1 - p).  Positions of [cur, nvalid) no selected match covers are literals;
 *     entry = wb + max(end of the last match, nvalid).
 *
 * Rule flags (F_*) each change one rule, so a test can show that a comparison with the kernel tells them apart.
 * Counters (what the member exercised, summed over its chunks) show that a comparison reached every rule. */
#include <stdint.h>
#include <string.h>

#ifdef __cplusplus
#define EXPORT extern "C"
#else
#define EXPORT
#endif

enum { CHUNK = 65536, PIECE = 4096, PHASE = 32768, PHASE_HIST = 1024, PRESEED = 2048, MAXM = 258, MINM = 4,
       MAXD = 32768, CAP = 32, HASH_BITS = 11, ENTRIES = 1 << HASH_BITS, EMPTY = 0xffff };

/* rule flags */
enum {
  F_PRESEED_2K = 1,   /* every piece but the first is pre-seeded with the full 2 KiB before it */
  F_LIMIT3 = 2,       /* a lane may match with only 3 bytes left before the piece end */
  F_TWO_ROUNDS = 4,   /* two doubling rounds: at most 4 selected matches per window */
  F_NO_EXIT_EXT = 8,  /* the window's last match is not extended past the lane cap */
  F_LOWEST = 16       /* same-entry stores of one instruction: the lowest position lands */
};

/* counter slots */
enum {
  C_MATCHES,          /* selected matches */
  C_COLLISIONS,       /* candidates in reach whose 4 bytes differ (a hash collision) */
  C_PRESEED_HITS,     /* selected matches whose source lies before the piece (in its pre-seed) */
  C_PRESEED_SHORT,    /* ... of the piece at 32768, whose pre-seed is 1 KiB */
  C_CAP_EXT,          /* windows whose last selected match reached the lane cap (the exit match) */
  C_M258,             /* selected 258-byte matches */
  C_LIMIT_CUT,        /* selected matches that end at the piece end although the bytes go on matching */
  C_SKIPPED,          /* windows skipped because a match covered them */
  C_WIN8,             /* windows with 8 selected matches */
  C_CONTESTED_STORES, /* (store instruction, entry) pairs written by 2 or more lanes */
  C_CONTESTED_READS,  /* probes whose candidate decides a match test and read an entry last written contested */
  /* per-window work, for tools/lz1_model.py */
  C_WINDOWS,          /* windows */
  C_ENTERED,          /* windows entered */
  C_VERIFIED,         /* lanes that pass the 4-byte check */
  C_EXT_STEPS_LANES,  /* 4-byte extension steps, summed over lanes */
  C_EXT_STEPS_WARP,   /* 4-byte extension steps, the maximum over the window's lanes */
  C_COUNT
};

static uint32_t rd32(const uint8_t *b) { return (uint32_t)b[0] | (uint32_t)b[1] << 8 | (uint32_t)b[2] << 16 | (uint32_t)b[3] << 24; }
static uint32_t lz_hash(uint32_t v) { return (v * 0x9E3779B1u) >> (32 - HASH_BITS); }

/* common prefix of a[0..] and b[0..], at most n */
static uint32_t prefix(const uint8_t *a, const uint8_t *b, uint32_t n) {
  uint32_t k = 0;
  while (k < n && a[k] == b[k]) k++;
  return k;
}

typedef struct {
  uint32_t *tok;
  uint64_t ntok, cap;
  uint64_t *cnt;
  int overflow;
} Out;

static void emit(Out *o, uint32_t t) {
  if (o->ntok < o->cap) o->tok[o->ntok] = t;
  else o->overflow = 1;
  o->ntok++;
}

typedef struct {
  uint16_t pos[ENTRIES];
  uint8_t contested[ENTRIES];   /* the entry's last write was contested */
} Table;

/* one store instruction: lanes p = base + l (l < 32) with ok[l] store position p to entry h[l] */
static void store32(Table *T, uint32_t base, const uint32_t *h, const int *ok, int lowest, uint64_t *cnt) {
  for (int l = 0; l < 32; l++) {
    if (!ok[l]) continue;
    int first = 1, n = 0;
    for (int j = 0; j < 32; j++)
      if (ok[j] && h[j] == h[l]) {
        if (j < l) first = 0;
        n++;
      }
    if (!first) continue;   /* each entry once, from its lowest lane */
    uint32_t win = base + (uint32_t)l;
    if (!lowest)
      for (int j = l + 1; j < 32; j++)
        if (ok[j] && h[j] == h[l]) win = base + (uint32_t)j;
    T->pos[h[l]] = (uint16_t)win;
    T->contested[h[l]] = n >= 2;
    if (n >= 2) cnt[C_CONTESTED_STORES]++;
  }
}

static void model_chunk(const uint8_t *B, uint32_t len, int mode, uint32_t flags, Out *o) {
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
    if (mode == 1) {
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
      if (mode == 1) {
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
          if (!(c[l] < p && p - c[l] <= MAXD)) continue;
          if (memcmp(B + c[l], B + p, 4) != 0) {
            cnt[C_COLLISIONS]++;
            continue;
          }
          cnt[C_VERIFIED]++;
          /* 4 bytes, then 4 more per step up to the lane cap; bytes past the chunk never match */
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

/* Parse one member: mode 1 is level 1, mode 0 the literals-only parse (level -2).  chunk_ntok[k] receives the
 * number of tokens of chunk k (room for max(1, ceil(n / 65536)) entries); counters has C_COUNT slots and is added
 * to.  Returns the total number of tokens, or -1 when `cap` is too small (nothing beyond cap is written). */
EXPORT int64_t lz1_model(const uint8_t *member, uint64_t n, int mode, uint32_t flags, uint32_t *tok, uint64_t cap,
                         uint32_t *chunk_ntok, uint64_t *counters) {
  Out o;
  memset(&o, 0, sizeof o);
  o.tok = tok;
  o.cap = cap;
  o.cnt = counters;
  const uint64_t nchunks = n == 0 ? 1 : (n + CHUNK - 1) / CHUNK;
  for (uint64_t k = 0; k < nchunks; k++) {
    const uint64_t before = o.ntok, c0 = k * CHUNK;
    model_chunk(member + c0, (uint32_t)(n - c0 < CHUNK ? n - c0 : CHUNK), mode, flags, &o);
    chunk_ntok[k] = (uint32_t)(o.ntok - before);
  }
  return o.overflow ? -1 : (int64_t)o.ntok;
}

EXPORT int lz1_counter_count(void) { return C_COUNT; }
