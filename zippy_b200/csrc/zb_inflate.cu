// zb_inflate.cu -- batched inflate for sm_90a: 8 lanes per compressed member, 4 members per
// warp decoded in lockstep, members pulled from a device work queue.
//
// Follows the behaviour (not the code) of the reference decoder:
//   format detect + wrappers : src/zippy.nim:100-165, src/zippy/gzip.nim:3-88
//   block loop               : src/zippy/inflate.nim:268-291
//   stored / fixed / dynamic : inflate.nim:252-266, 104-171
//   symbol loop + back-copy  : inflate.nim:173-250
//   canonical decode         : inflate.nim:24-102 (same accept/reject set: over-subscribed
//                              length sets are rejected, incomplete ones accepted, an
//                              undecodable code is an error)
// GPU formulation (DESIGN.md section 4): a DEFLATE stream is one long
// dependency chain, so the kernel is built around (a) keeping that chain short -- a register bit
// window per member, table entries that carry the number of bits a token occupies, two literals
// per slot -- (b) making every warp instruction advance four members at once (a predicated
// token loop that all groups of a warp run together) and (c) doing everything that is not on
// the chain lane-parallel afterwards (32 raw tokens per member are validated, placed by a prefix
// sum and copied one lane per token).  Large members are split at sync markers into segments
// that run through the same kernel in parallel (zb_api.cu: inflate_big_members).
#include <type_traits>

#include <algorithm>

#include "zb_device.cuh"
#include "zb_kernels.h"
#include "zb_resolve.h"
#include "zb_wrapper.h"

#ifndef INF_G
#define INF_G 8                       // lanes per member; 32 / INF_G members are decoded per warp
#endif
#ifndef INF_WARPS
#define INF_WARPS 4
#endif
#define INF_THREADS (INF_WARPS * 32)
#define INF_GROUPS (INF_THREADS / INF_G)
#define FULL_MASK 0xffffffffu
#ifndef INF_SPLIT_LONG
#define INF_SPLIT_LONG 0   // 1: of more than 32 bits are consumed in two steps by the rare path (slower: the test sits on the bit-position chain)
#endif

// A "group" is INF_G consecutive lanes that decode one member together; every lane of a group
// keeps the same decoder state, group collectives are restricted to the group's own lanes.  The
// 32 / INF_G groups of a warp run the symbol loop in LOCKSTEP: one iteration decodes one token for
// every group with the literal / match paths predicated instead of branched, so a warp instruction
// advances 32 / INF_G members at once.  (A first attempt at two members per warp with a branching
// token loop was slower than one member per warp: the halves never reconverged.)
__device__ __forceinline__ int g_lane() { return (int)(threadIdx.x & (INF_G - 1)); }
__device__ __forceinline__ uint32_t g_shift() { return threadIdx.x & 31u & ~(uint32_t)(INF_G - 1); }
__device__ __forceinline__ uint32_t g_mask() { return (INF_G == 32 ? 0xffffffffu : ((1u << INF_G) - 1u)) << g_shift(); }
__device__ __forceinline__ uint32_t g_shfl(uint32_t v, int idx) { return __shfl_sync(g_mask(), v, idx, INF_G); }
__device__ __forceinline__ uint32_t g_ballot(bool p) {
  return (__ballot_sync(g_mask(), p) >> g_shift()) & (INF_G == 32 ? 0xffffffffu : ((1u << INF_G) - 1u));
}
__device__ __forceinline__ uint32_t g_match_any(uint32_t v) { return __match_any_sync(g_mask(), v) >> g_shift(); }
__device__ __forceinline__ void g_sync() { __syncwarp(g_mask()); }
// Table sizes trade slow-path decodes against occupancy: the kernel is bound by the latency of
// the per-token dependency chain, so warps per SM matter more than table hits: 9 + 8 bits leave room
// for 20 warps per SM, 10 + 9 bits for 12.
#ifndef LL_BITS
#define LL_BITS 9    // literal/length codes up to this long decode with one table lookup
#endif
#ifndef D_BITS
#define D_BITS 8     // same for distance codes (>= 7: the table also serves the code-length code)
#endif

struct GroupSmem {
  uint16_t lut_ll[1 << LL_BITS];  // symbol | code length << 9; 0 = longer code or no code: slow path
  uint16_t lut_d[1 << D_BITS];
  uint16_t syms_ll[288];          // symbols sorted by (length, symbol) for the canonical slow path
  uint16_t syms_d[32];
  uint8_t lens[320];              // code lengths of the current block (lit/len then distance)
  uint16_t cnt[16];               // per-length counts / running ranks while building
  uint16_t first[2][16];          // canonical ranges per code length: [0] literal/length, [1] distance
  uint16_t count[2][16];          //   (and the code-length code while a dynamic header is read)
  uint16_t offs[2][16];
};
static_assert(sizeof(GroupSmem) % 16 == 0, "group tables must keep 16-byte alignment");

// Bit window of one member (identical in every lane of its group).  The compressed bytes are
// viewed as 32-bit words from `gbase`; lane j of the group holds word j of two consecutive
// "lines" (INF_G words each), refilled by one coalesced load per line; the three words at the
// read position live in registers (w0, w1, w2) and the next two are fetched by shuffle while
// the current token is being decoded, so consuming up to 48 bits per token never waits on memory.
struct BitReader {
  const uint32_t *gbase;  // member start rounded down to 4 bytes
  uint32_t nwords;        // words that contain member bytes (beyond: zeros)
  uint32_t last_mask;     // member bytes of word nwords - 1: the bytes after the member read as zero too
  uint32_t cur, nxt;     // lane-held words of the line that holds word wi + 3, and of the next line
  uint32_t w0, w1, w2;    // words wi, wi + 1, wi + 2
  uint32_t wi;
  uint32_t bo;            // next unread bit inside w0 (0..31)
  uint64_t end_bit;       // absolute bit (from gbase) one past the member's last byte
  bool overrun;           // the reader is far past the end: whatever is being decoded is garbage
};

// Bits past the member's last byte read as zero, as in the reference's bit reader
// (bitstreams.nim:22-48): a verdict that reads them (extra bits of a truncated token or repeat code) must
// not depend on the bytes that follow the member in the batch buffer.
__device__ __forceinline__ uint32_t br_word(const BitReader &b, uint32_t idx) {
  if (idx >= b.nwords) return 0u;
  const uint32_t v = __ldcg(b.gbase + idx);  // L2 only: every word is read once, and with a gated queue the
                                             // line may hold bytes of a member whose copy-in has not landed yet
  return idx + 1u == b.nwords ? v & b.last_mask : v;
}
__device__ __forceinline__ uint32_t br_tail_mask(uint64_t end_byte) {  // end_byte: one past the last byte, from gbase
  const uint32_t r = (uint32_t)end_byte & 3u;
  return r ? (1u << (8u * r)) - 1u : 0xffffffffu;
}
__device__ __forceinline__ uint32_t br_load_line(const BitReader &b, uint32_t line) {
  return br_word(b, line * (uint32_t)INF_G + (uint32_t)g_lane());
}
__device__ __forceinline__ uint64_t br_consumed_abs(const BitReader &b) { return (uint64_t)b.wi * 32ull + b.bo; }
__device__ __forceinline__ bool br_past_end(const BitReader &b) { return br_consumed_abs(b) > b.end_bit; }
// position the reader at byte `byte_off` of the member (shift0 = member start & 3)
__device__ __forceinline__ void br_seek(BitReader &b, uint32_t shift0, uint64_t byte_off) {
  uint64_t abit = (shift0 + byte_off) * 8ull;
  b.wi = (uint32_t)(abit >> 5);
  b.bo = (uint32_t)(abit & 31u);
  b.w0 = br_word(b, b.wi);
  b.w1 = br_word(b, b.wi + 1u);
  b.w2 = br_word(b, b.wi + 2u);
  const uint32_t line = (b.wi + 3u) / (uint32_t)INF_G;
  b.cur = br_load_line(b, line);
  b.nxt = br_load_line(b, line + 1u);
}
// word wi + 3 has just moved into a new line
__device__ __forceinline__ void br_advance_line(BitReader &b) {
  b.cur = b.nxt;
  b.nxt = br_load_line(b, (b.wi + 3u) / (uint32_t)INF_G + 1u);
  // bits past the end read as zero; a reader that is well past the end can only be decoding
  // garbage: flag it here so that no decode loop runs away (checked by the callers)
  if (b.wi > (uint32_t)((b.end_bit + 64ull) >> 5)) b.overrun = true;
}
// Consume n bits.  LOCKSTEP: every lane of the warp executes the call together (the symbol
// loop), so the shuffle can name the full warp; groups with n == 0 keep their state; n <= 32
// there (longer tokens are split by the caller).  Otherwise n <= 48.
template <bool LOCKSTEP>
__device__ __forceinline__ uint32_t br_skip(BitReader &b, uint32_t n) {
  // shfl takes the source lane modulo the width: lane (wi + 3) % INF_G of the group holds word wi + 3
  const uint32_t n0 = LOCKSTEP ? __shfl_sync(FULL_MASK, b.cur, (int)(b.wi + 3u), INF_G) : g_shfl(b.cur, (int)(b.wi + 3u));
  const uint32_t pos = b.bo + n;
  const uint32_t k = pos >> 5;  // whole words consumed: 0, 1 or (tokens longer than 32 bits) 2
  // the 32 bits at the new position, from the window as it is (valid for pos < 64): lets the
  // next token start without waiting for the window registers to move
  const uint32_t peek = (pos & 32u) ? __funnelshift_r(b.w1, b.w2, pos) : __funnelshift_r(b.w0, b.w1, pos);
  b.bo = pos & 31u;
  const bool k1 = k != 0u;
  b.w0 = k1 ? b.w1 : b.w0;
  b.w1 = k1 ? b.w2 : b.w1;
  b.w2 = k1 ? n0 : b.w2;
  b.wi += k1 ? 1u : 0u;
  if (k1 && ((b.wi + 3u) & (uint32_t)(INF_G - 1)) == 0u) br_advance_line(b);
  if ((!LOCKSTEP || !INF_SPLIT_LONG) && k >= 2u) {  // rare
    const uint32_t n1 = g_shfl(b.cur, (int)(b.wi + 3u));
    b.w0 = b.w1;
    b.w1 = b.w2;
    b.w2 = n1;
    b.wi++;
    if (((b.wi + 3u) & (uint32_t)(INF_G - 1)) == 0u) br_advance_line(b);
    return __funnelshift_r(b.w0, b.w1, b.bo);
  }
  return peek;
}
__device__ __forceinline__ uint32_t br_peek(const BitReader &b) { return __funnelshift_r(b.w0, b.w1, b.bo); }
__device__ __forceinline__ uint32_t br_take(BitReader &b, int n) {  // n <= 16
  uint32_t v = br_peek(b) & ((1u << n) - 1u);
  br_skip<false>(b, (uint32_t)n);
  return v;
}
// base + 2 * idx in one instruction (the address of a 16-bit table entry)
__device__ __forceinline__ uint32_t lut_addr(uint32_t base, uint32_t idx) {
  uint32_t a;
  asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(a) : "r"(idx), "r"(base));
  return a;
}
// shared-memory reads by 32-bit shared address (the decode tables in the symbol loop)
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// Build the decode state from n code lengths (inflate.nim:24-65 initHuffman): the per-length
// canonical ranges (for the lane-parallel slow path), the sorted symbols, and a direct lookup
// table for codes of at most lut_bits.  Table entries (0 = no code this short: slow path):
//   KIND 0 (code-length code): symbol | len << 9
//   KIND 1 (literal/length)  : symbol | (len + extra bits of a length symbol) << 11
//   KIND 2 (distance)        : symbol | (len + extra bits) << 11
// so the number of bits a token occupies is one shift away from the table entries and nothing
// else (base values, the split of code and extra bits) sits on the bit-position dependency chain.
// Returns false for an over-subscribed set (inflate.nim:32-34, 45-46).
template <int KIND>
__device__ __forceinline__ bool build_tree(const uint8_t *lens, int n, uint16_t *syms, uint16_t *lut, int lut_bits,
                                           GroupSmem *gs, int which) {
  const int lane = g_lane();
  for (int i = lane; i < 16; i += INF_G) gs->cnt[i] = 0;
  {
    uint4 z = make_uint4(0u, 0u, 0u, 0u);
    uint4 *l4 = reinterpret_cast<uint4 *>(lut);
    for (int i = lane; i < ((1 << lut_bits) * 2) / 16; i += INF_G) l4[i] = z;
  }
  g_sync();
  for (int base = 0; base < n; base += INF_G) {
    int s = base + lane;
    uint32_t l = s < n ? lens[s] : 0u;
    uint32_t grp = g_match_any(l);
    if (l && lane == __ffs((int)grp) - 1) gs->cnt[l] = (uint16_t)(gs->cnt[l] + __popc(grp));
    g_sync();
  }
  // per-length first code / first slot (all lanes compute the same recurrence)
  bool ok = true;
  uint32_t code = 0, k = 0;
  for (int i = 1; i < 16; i++) {
    uint32_t c = gs->cnt[i];
    if (lane == 0) {
      gs->first[which][i] = (uint16_t)code;
      gs->count[which][i] = (uint16_t)c;
      gs->offs[which][i] = (uint16_t)k;
    }
    code += c;
    if (c > 0 && code - 1 >= (1u << i)) ok = false;
    code <<= 1;
    k += c;
  }
  g_sync();
  for (int i = lane; i < 16; i += INF_G) gs->cnt[i] = 0;  // becomes the running rank per length
  if (lane == 0) gs->count[which][0] = 0;
  g_sync();
  if (!ok) return false;
  for (int base = 0; base < n; base += INF_G) {
    int s = base + lane;
    uint32_t l = s < n ? lens[s] : 0u;
    uint32_t grp = g_match_any(l);
    if (l) {
      uint32_t rank = gs->cnt[l] + (uint32_t)__popc(grp & ((1u << lane) - 1u));
      syms[(uint32_t)gs->offs[which][l] + rank] = (uint16_t)s;
      if ((int)l <= lut_bits) {
        uint32_t c = (uint32_t)gs->first[which][l] + rank;   // canonical code, MSB first
        uint32_t rev = __brev(c) >> (32 - l);                // as it appears in the LSB-first stream
        uint32_t e = (uint32_t)s | (l << 9);
        if (KIND == 1) e = (uint32_t)s | ((l + ((s > 256 && s < 286) ? (uint32_t)zb_len_extra_bits(s - 257) : 0u)) << 11);
        if (KIND == 2) e = (uint32_t)s | ((l + (s < 30 ? (uint32_t)zb_dist_extra_bits(s) : 0u)) << 11);
        for (uint32_t idx = rev; idx < (1u << lut_bits); idx += (1u << l)) lut[idx] = (uint16_t)e;
      }
    }
    g_sync();
    if (l && lane == __ffs((int)grp) - 1) gs->cnt[l] = (uint16_t)(gs->cnt[l] + __popc(grp));
    g_sync();
  }
  return true;
}

// Lane-parallel canonical decode of the code at the low end of x (codes longer than the lookup
// table, and the "no code matches" case, which returns 0xffff with L = 0: inflate.nim:77-82).
// Lane j tests the code lengths j, j + INF_G, ...; a ballot picks the shortest that matches.
__device__ __forceinline__ uint32_t decode_slow(uint32_t x, const GroupSmem *gs, int which, const uint16_t *syms,
                                                uint32_t &L_out) {
  const int lane = g_lane();
  const uint32_t rev = __brev(x);
  for (int base = 0; base < 16; base += INF_G) {
    const int L = base + lane;
    const uint32_t code = (L >= 1 && L < 16) ? (rev >> (32 - L)) : 0u;
    const uint32_t rel = code - (uint32_t)gs->first[which][L & 15];
    const bool h = L >= 1 && L < 16 && rel < (uint32_t)gs->count[which][L & 15];
    const uint32_t hit = g_ballot(h);
    if (hit) {
      const int j = __ffs((int)hit) - 1;
      const uint32_t idx = g_shfl((uint32_t)gs->offs[which][L & 15] + rel, j);
      L_out = (uint32_t)(base + j);
      return syms[idx];
    }
  }
  L_out = 0;
  return 0xffffu;
}
// One symbol of the code-length code (dynamic header).
__device__ __forceinline__ uint32_t decode_clc(BitReader &b, const GroupSmem *gs) {
  const uint32_t x = br_peek(b);
  const uint32_t e = gs->lut_d[x & 127u];
  uint32_t l = e >> 9, sym = e & 511u;
  if (l == 0) sym = decode_slow(x, gs, 1, gs->syms_d, l);
  br_skip<false>(b, l);
  return sym;
}

// Validate and materialise a batch of up to 32 decoded tokens of one group.  Token k of the batch
// sits in lane k % INF_G, slot k / INF_G, still "raw" as the symbol loop decoded it:
//   ta = symbol (9 bits) | length extra value << 9 | second table entry << 14
//   tb = distance extra value (13 bits) | reader position after the token << 13
// The second table entry is the distance entry (symbol | (code + extra bits) << 11) after a
// length symbol; after a literal it is the literal/length entry of the NEXT symbol, and
// when that is a literal too (symbol < 256, code length != 0) the slot holds both bytes.
// Everything that does not feed the bit position is done HERE, one lane per token instead of
// redundantly by the whole group: base values (RFC 1951 3.2.5), the checks of inflate.nim:203,
// 212, 224 (length symbol >= 29, distance symbol >= 30, distance > bytes produced) and the
// capacity check.  A group prefix sum of the lengths places every token.  Literals and short
// matches whose source lies wholly before the batch are copied by their own lane, all in parallel
// (loads first, then stores: the sources cannot alias anything written here); matches that read
// bytes produced inside the batch, and long ones, follow in stream order, each copied by the
// whole group (reads only touch finished output: i % dist).
// Returns 0, or 2 (invalid token) / 3 (out of room) for the first offending token in stream order
// (bad_back: how many bits before the token's end its end-of-input verdict is taken),
// whose index is stored to bad_k; only the tokens before it are written and counted in op.
#define INF_ROUNDS (32 / INF_G)
#define INF_LONG_MATCH 24u
// OutT is uint8_t, or uint16_t when a segment of a large member is decoded without its window
// (zb_api.cu: speculative segments): the 32768 elements in front of `out` then hold marker symbols
// 0x8000 | k standing for "byte k of the unknown window", copies move markers like literals, and `win`
// (0 or 32768) is how far before its own start the segment may reach.
// DICT (byte output only): a member decoded against a preset dictionary.  `win` is then the window length and wend
// points just past the window W: output position p < 0 (relative to `out`) is the byte wend[p].  Every copy reads
// through copy_src, so a match may lie in W, in the output, or straddle the two.
template <bool DICT, typename OutT>
__device__ __forceinline__ OutT copy_src(const OutT *out, const uint8_t *wend, int64_t p) {
  if (DICT && p < 0) return (OutT)wend[p];
  return out[p];
}
template <bool COUNT_ONLY, typename OutT, bool DICT = false>
__device__ __forceinline__ int flush_tokens(OutT *out, uint32_t &op, uint32_t cap, uint32_t win,
                                            const uint32_t (&ta)[INF_ROUNDS], const uint32_t (&tb)[INF_ROUNDS],
                                            uint32_t ntok, uint32_t len_addr, uint32_t dist_addr, uint32_t &bad_k,
                                            uint32_t &bad_back, const uint8_t *wend = nullptr) {
  const int lane = g_lane();
  const uint32_t gsel = INF_G == 32 ? 0xffffffffu : ((1u << INF_G) - 1u);
  const uint32_t batch_op = op;
  uint32_t len[INF_ROUNDS], rel[INF_ROUNDS], dist[INF_ROUNDS];
  bool is_m[INF_ROUNDS], dep[INF_ROUNDS];
  uint32_t base = 0, evm[INF_ROUNDS], badm[INF_ROUNDS];
  bool any_ev = false;
#pragma unroll
  for (int r = 0; r < INF_ROUNDS; r++) {
    const bool act = (uint32_t)(r * INF_G + lane) < ntok;
    const uint32_t sym = ta[r] & 511u;
    const uint32_t lidx = min(sym - 257u, 31u);
    const uint32_t e2 = ta[r] >> 14;
    const uint32_t dsym = e2 & 31u;
    const bool two = (e2 & 511u) < 256u && (e2 >> 11) != 0u;  // (only looked at for a literal)
    is_m[r] = act && sym > 256u;
    len[r] = act ? (is_m[r] ? (lds_u32(len_addr + lidx * 4u) & 0xffffu) + ((ta[r] >> 9) & 31u) : (two ? 2u : 1u)) : 0u;
    dist[r] = (lds_u32(dist_addr + dsym * 4u) & 0xffffu) + (tb[r] & 0x1fffu);
    uint32_t incl = len[r];
#pragma unroll
    for (int o = 1; o < INF_G; o <<= 1) {  // the whole warp is here together: full-mask shuffles
      uint32_t t = __shfl_up_sync(FULL_MASK, incl, o, INF_G);
      if (lane >= o) incl += t;
    }
    rel[r] = base + incl - len[r];  // output offset inside the batch
    base += __shfl_sync(FULL_MASK, incl, INF_G - 1, INF_G);
    const bool bad = is_m[r] && (lidx >= 29u || dsym >= 30u || dist[r] > batch_op + rel[r] + win);
    const bool noroom = act && rel[r] + len[r] > cap - batch_op;
    badm[r] = (__ballot_sync(FULL_MASK, bad) >> g_shift()) & gsel;
    evm[r] = (__ballot_sync(FULL_MASK, bad || noroom) >> g_shift()) & gsel;
    any_ev = any_ev || evm[r] != 0u;
  }
  int ev = 0;
  uint32_t n_ok = ntok, total = base;
  if (any_ev) {  // rare: cut the batch at the first offending token
#pragma unroll
    for (int r = INF_ROUNDS - 1; r >= 0; r--) {
      if (evm[r]) {
        const int j = __ffs((int)evm[r]) - 1;
        n_ok = (uint32_t)(r * INF_G + j);
        ev = ((badm[r] >> j) & 1u) ? 2 : 3;
        total = g_shfl(rel[r], j);
        // a distance symbol >= 30 is judged before the end of the input is (inflate.nim:212-213): the
        // caller checks the end where the literal/length code ends, this many bits before the token's end
        const uint32_t li = (ta[r] & 511u) - 257u;
        const uint32_t back = (li < 29u && ((ta[r] >> 14) & 31u) >= 30u) ? (ta[r] >> 25) + (lds_u32(len_addr + li * 4u) >> 16) : 0u;
        bad_back = g_shfl(back, j);
      }
    }
    bad_k = n_ok;
#pragma unroll
    for (int r = 0; r < INF_ROUNDS; r++) {
      if ((uint32_t)(r * INF_G + lane) >= n_ok) {
        len[r] = 0;
        is_m[r] = false;
      }
    }
  }
  op = batch_op + total;
  if (COUNT_ONLY) return ev;
  __syncwarp();  // stores of earlier batches are visible to every lane from here on
  OutT *const bout = out + batch_op;
  // parallel part, 4 bytes per token and pass
  uint32_t more = 0;
#pragma unroll
  for (int r = 0; r < INF_ROUNDS; r++) {
    dep[r] = is_m[r] && (dist[r] < rel[r] + len[r] || len[r] > INF_LONG_MATCH);
    if (len[r] != 0u && !is_m[r]) {
      bout[rel[r]] = (OutT)(uint8_t)ta[r];
      if (len[r] == 2u) bout[rel[r] + 1u] = (OutT)(uint8_t)(ta[r] >> 14);
    }
    if (is_m[r] && !dep[r] && len[r] > 4u) more |= 1u << r;
  }
  {
    OutT v[INF_ROUNDS][4];
#pragma unroll
    for (int r = 0; r < INF_ROUNDS; r++) {
      const OutT *from = bout + rel[r] - dist[r];
      const bool go = is_m[r] && !dep[r];
      if (DICT) {
        const int64_t p0 = (int64_t)batch_op + rel[r] - dist[r];
#pragma unroll
        for (int k = 0; k < 4; k++) v[r][k] = (go && (uint32_t)k < len[r]) ? copy_src<DICT>(out, wend, p0 + k) : (OutT)0;
      } else {
#pragma unroll
        for (int k = 0; k < 4; k++) v[r][k] = (go && (uint32_t)k < len[r]) ? from[k] : (OutT)0;
      }
    }
#pragma unroll
    for (int r = 0; r < INF_ROUNDS; r++) {
      const bool go = is_m[r] && !dep[r];
#pragma unroll
      for (int k = 0; k < 4; k++)
        if (go && (uint32_t)k < len[r]) bout[rel[r] + k] = v[r][k];
    }
  }
  if (more) {
#pragma unroll
    for (int r = 0; r < INF_ROUNDS; r++) {
      if (more & (1u << r)) {
        OutT *to = bout + rel[r];
        const OutT *from = to - dist[r];
        if (DICT) {
          const int64_t p0 = (int64_t)batch_op + rel[r] - dist[r];
          for (uint32_t k = 4; k < len[r]; k++) to[k] = copy_src<DICT>(out, wend, p0 + k);
        } else {
          for (uint32_t k = 4; k < len[r]; k += 4) {
            OutT c0 = from[k], c1 = k + 1 < len[r] ? from[k + 1] : (OutT)0, c2 = k + 2 < len[r] ? from[k + 2] : (OutT)0,
                 c3 = k + 3 < len[r] ? from[k + 3] : (OutT)0;
            to[k] = c0;
            if (k + 1 < len[r]) to[k + 1] = c1;
            if (k + 2 < len[r]) to[k + 2] = c2;
            if (k + 3 < len[r]) to[k + 3] = c3;
          }
        }
      }
    }
  }
  // ordered part
#pragma unroll
  for (int r = 0; r < INF_ROUNDS; r++) {
    uint32_t depmask = (__ballot_sync(FULL_MASK, dep[r]) >> g_shift()) & gsel;
    while (depmask) {
      const int j = __ffs((int)depmask) - 1;
      depmask &= depmask - 1;
      const uint32_t rj = g_shfl(rel[r], j), lj = g_shfl(len[r], j);
      const uint32_t dj = g_shfl(dist[r], j);
      g_sync();
      OutT *tj = bout + rj;
      const OutT *fj = tj - dj;
      if (DICT) {
        const int64_t p0 = (int64_t)batch_op + rj - dj;
        for (uint32_t i = (uint32_t)lane; i < lj; i += INF_G) tj[i] = copy_src<DICT>(out, wend, p0 + (dj >= lj ? i : i % dj));
      } else if (dj >= lj) {
        for (uint32_t i = (uint32_t)lane; i < lj; i += INF_G) tj[i] = fj[i];
      } else {
        for (uint32_t i = (uint32_t)lane; i < lj; i += INF_G) tj[i] = fj[i % dj];
      }
    }
  }
  return ev;
}

// ---- per-group decoder state (identical in every lane of the group) ----
enum { ST_FETCH = 0, ST_BLOCK = 1, ST_SYMS = 2, ST_EXIT = 3 };
// ---- gated queue (ZbInflateWork::gate_*) ----
__device__ __forceinline__ uint32_t gate_load(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t gate_clock() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// every lane of the group calls this after the member's last output store
__device__ __forceinline__ void gate_member_done(const ZbInflateWork &w, uint32_t gate) {
  if (!w.gate_done) return;
  __threadfence();  // this lane's output bytes are visible device-wide ...
  g_sync();
  if (g_lane() == 0) atomicAdd(w.gate_done + gate, 1u);  // ... before the count that releases the group's copy-out
}

template <typename OutT>
struct Grp {
  BitReader b;
  const uint8_t *src;   // member bytes
  uint64_t len;
  OutT *out;
  uint32_t shift0, cap, op, idx, kind, expect;
  uint32_t win;         // elements in front of `out` a back-reference may reach (speculative segments: 32768)
  uint32_t gate;        // gated queue: the copy-in group of the member in hand
  uint32_t ready_seen;  // gated queue: copy-in groups this group knows to have landed
  int st;
  bool final_block;
};

// Read one block header (inflate.nim:273-289, 104-171).  Stored blocks are copied here.
// Returns BLK_SYMS when the decode tables are ready for the symbol loop, BLK_DONE when the block
// is already complete (stored), or a (positive) ZB_ERR_*.
enum { BLK_SYMS = -1, BLK_DONE = -2 };
template <bool COUNT_ONLY, typename OutT>
__device__ __forceinline__ int begin_block(Grp<OutT> &g, GroupSmem *gs) {
  const int lane = g_lane();
  const uint8_t clcl_order[19] = ZB_CLCL_ORDER;
  BitReader &b = g.b;
  uint32_t bfinal = br_take(b, 1);
  uint32_t btype = br_take(b, 2);
  if (br_past_end(b)) return ZB_ERR_END_OF_BUFFER;
  if (bfinal) g.final_block = true;
  if (btype == 0) {
    // ---- stored (inflate.nim:252-266) ----
    br_skip<false>(b, (8u - (b.bo & 7u)) & 7u);
    uint32_t l = br_take(b, 16);
    uint32_t nl = br_take(b, 16);
    if (br_past_end(b)) return ZB_ERR_END_OF_BUFFER;
    if (l + nl != 65535u) return ZB_ERR_UNCOMPRESS;
    if (l > 0) {
      uint64_t byte_pos = (br_consumed_abs(b) >> 3) - g.shift0;
      if (byte_pos + l > g.len) return ZB_ERR_END_OF_BUFFER;
      if (l > g.cap - g.op) return ZB_ERR_DST_TOO_SMALL;
      if (!COUNT_ONLY)
        for (uint32_t i = (uint32_t)lane; i < l; i += INF_G) g.out[g.op + i] = (OutT)g.src[byte_pos + i];
      g.op += l;
      br_seek(b, g.shift0, byte_pos + l);
    }
    return BLK_DONE;
  }
  if (btype == 3) return ZB_ERR_BLOCK_HEADER;
  int hlit, hdist;
  if (btype == 1) {
    // ---- fixed codes (inflate.nim:111-113) ----
    for (int i = lane; i < 320; i += INF_G) gs->lens[i] = (uint8_t)(i < 288 ? zb_fixed_ll_len(i) : 5);
    hlit = 288;
    hdist = 30;
    g_sync();
  } else {
    // ---- dynamic header (inflate.nim:115-171) ----
    hlit = (int)br_take(b, 5) + 257;
    hdist = (int)br_take(b, 5) + 1;
    int hclen = (int)br_take(b, 4) + 4;
    if (hlit > ZB_NUM_LITLEN) return ZB_ERR_UNCOMPRESS;
    if (hdist > ZB_NUM_DIST) return ZB_ERR_UNCOMPRESS;
    for (int i = lane; i < 19; i += INF_G) gs->lens[i] = 0;
    g_sync();
    for (int i = 0; i < hclen; i++) {
      uint32_t v = br_take(b, 3);
      if (lane == 0) gs->lens[clcl_order[i]] = (uint8_t)v;
    }
    g_sync();
    if (!build_tree<0>(gs->lens, 19, gs->syms_d, gs->lut_d, 7, gs, 1)) return ZB_ERR_UNCOMPRESS;
    g_sync();
    // the code-length code now lives in syms_d / lut_d; lens[] is rewritten with the
    // unpacked literal/length + distance code lengths.
    int i = 0;
    const int total = hlit + hdist;
    uint32_t prev = 0;
    while (i != total) {
      uint32_t sym = decode_clc(b, gs);
      // inflate.nim:135-168 order: a symbol that ends past the input is the end of the buffer before
      // anything else; the repeat count read after it is not checked until the next symbol (or the
      // symbol loop), so a repeat that overshoots hlit + hdist first is an invalid header
      if (br_past_end(b)) return ZB_ERR_END_OF_BUFFER;
      if (sym <= 15) {
        if (lane == 0) gs->lens[i] = (uint8_t)sym;
        prev = sym;
        i++;
      } else if (sym == 16) {
        if (i == 0) return ZB_ERR_UNCOMPRESS;
        int rep = (int)br_take(b, 2) + 3;
        if (i + rep > 320) return ZB_ERR_UNCOMPRESS;
        for (int j = lane; j < rep; j += INF_G) gs->lens[i + j] = (uint8_t)prev;
        i += rep;
      } else if (sym == 17) {
        int rep = (int)br_take(b, 3) + 3;
        for (int j = lane; j < rep && i + j < 320; j += INF_G) gs->lens[i + j] = 0;
        i += rep;
        prev = 0;
      } else if (sym == 18) {
        int rep = (int)br_take(b, 7) + 11;
        for (int j = lane; j < rep && i + j < 320; j += INF_G) gs->lens[i + j] = 0;
        i += rep;
        prev = 0;
      } else {
        return ZB_ERR_INVALID_SYMBOL;  // also the undecodable-code case (0xffff)
      }
      if (i > total) return ZB_ERR_UNCOMPRESS;
    }
    g_sync();
  }
  if (!build_tree<1>(gs->lens, hlit, gs->syms_ll, gs->lut_ll, LL_BITS, gs, 0)) return ZB_ERR_UNCOMPRESS;
  if (!build_tree<2>(gs->lens + hlit, hdist, gs->syms_d, gs->lut_d, D_BITS, gs, 1)) return ZB_ERR_UNCOMPRESS;
  g_sync();
  // the last repeat count of a dynamic header may have run past the input: the reference builds the
  // codes first (an over-subscribed set is an invalid header) and stops at the first symbol after
  if (br_past_end(b)) return ZB_ERR_END_OF_BUFFER;
  return BLK_SYMS;
}

// The symbol loop (inflate.nim:173-250) for all groups of the warp at once.  Every iteration
// decodes ONE token per decoding group; the match path is computed unconditionally and
// selected, so the groups stay converged whatever mix of literals and matches they see.  The
// bit position of the next token depends only on the two table entries (code length + extra
// bit count are both in the entry), which keeps the loop-carried dependency short; the loop
// itself only extracts the raw fields, flush_tokens turns them into bytes (and finds invalid
// tokens) one lane per token.  32 tokens per group are collected (token k in lane k % INF_G,
// slot k / INF_G) and then flushed; a group that reaches the end of its block idles until the
// batch ends, the loop stops, and the caller resolves the event.
// Returns 0 (another group stopped the loop), 1 (end of block) or 100 + ZB_ERR_*.
template <bool COUNT_ONLY, typename OutT, bool DICT = false>
__device__ __forceinline__ int symbol_loop(Grp<OutT> &g, const GroupSmem *gs, uint32_t tab_addr, const uint8_t *wend = nullptr) {
  const int lane = g_lane();
  bool act = g.st == ST_SYMS;
  BitReader &b = g.b;
  uint32_t op = g.op;
  // 32-bit shared addresses of this group's tables and of the base-value tables
  const uint32_t ll_addr = (uint32_t)__cvta_generic_to_shared(gs->lut_ll);
  const uint32_t d_addr = (uint32_t)__cvta_generic_to_shared(gs->lut_d);
  uint32_t len_addr = tab_addr;
  asm volatile("" : "+r"(len_addr));  // keep the address in a register (else it is recomputed from %cluster_ctaid per use)
  const uint32_t dist_addr = len_addr + 128u;
  const bool act0 = act;
  int ev = 0;
  for (;;) {
    // token k of the batch: lane k % INF_G, slot k / INF_G, two registers (see flush_tokens)
    uint32_t ta[INF_ROUNDS], tb[INF_ROUNDS];
    uint32_t ntok = 0;
    uint32_t x1 = br_peek(b);  // the 32 bits at the read position, carried from token to token
#pragma unroll
    for (int r = 0; r < INF_ROUNDS; r++) {
      ta[r] = 0;
      tb[r] = 0;
#pragma unroll 1
      for (int j = 0; j < INF_G; j++) {
        const uint32_t bo0 = b.bo;
        const uint32_t e = lds_u16(lut_addr(ll_addr, x1 & ((1u << LL_BITS) - 1u)));
        uint32_t sym = e & 511u, s1 = e >> 11;  // s1: code + extra bits of this symbol
        uint32_t p2 = bo0 + s1;                 // <= 31 + 20
        uint32_t x2 = (p2 & 32u) ? __funnelshift_r(b.w1, b.w2, p2) : __funnelshift_r(b.w0, b.w1, p2);
        // second lookup: the distance table after a length symbol; after a literal, the
        // literal/length table again -- two literals in a row leave as ONE token slot
        const bool lit1 = sym < 256u;
        uint32_t e2 = lds_u16(lut_addr(lit1 ? ll_addr : d_addr, x2 & (lit1 ? ((1u << LL_BITS) - 1u) : ((1u << D_BITS) - 1u))));
        uint32_t s2 = e2 >> 11;  // bits of the distance (code + extra), or of the second literal
        const bool pair = act && lit1 && s1 != 0u && s2 != 0u && (e2 & 511u) < 256u;
        bool want_d = act && (sym - 257u) < 29u;
        if (act && (s1 == 0u || (want_d && s2 == 0u))) {
          // rare: a code longer than its lookup table (or no code at all)
          if (s1 == 0u) {
            uint32_t l;
            sym = decode_slow(x1, gs, 0, gs->syms_ll, l);
            sym = l ? sym : 287u;  // no code: an invalid length symbol
            const uint32_t lidx = sym - 257u;
            s1 = l + (lidx < 29u ? (lds_u32(len_addr + lidx * 4u) >> 16) : 0u);
            want_d = lidx < 29u;
            p2 = bo0 + s1;
            x2 = (p2 & 32u) ? __funnelshift_r(b.w1, b.w2, p2) : __funnelshift_r(b.w0, b.w1, p2);
            e2 = want_d ? lds_u16(lut_addr(d_addr, x2 & ((1u << D_BITS) - 1u))) : 0u;  // 0: never a literal pair
            s2 = e2 >> 11;
          }
          if (want_d && s2 == 0u) {
            uint32_t l2;
            uint32_t dsym = decode_slow(x2, gs, 1, gs->syms_d, l2);
            dsym = l2 ? dsym : 31u;  // no code: an invalid distance symbol
            s2 = l2 + (dsym < 30u ? (lds_u32(dist_addr + dsym * 4u) >> 16) : 0u);
            e2 = dsym | (s2 << 11);
          }
        }
        const uint32_t adv = s1 + ((want_d || pair) ? s2 : 0u);
        const uint32_t x1n = br_skip<true>(b, act ? adv : 0u);
        // off the bit-position chain: the extra-bit values
        const uint32_t ext = want_d ? (lds_u32(len_addr + (sym - 257u) * 4u) >> 16) : 0u;
        const uint32_t dext = lds_u32(dist_addr + (e2 & 31u) * 4u) >> 16;
        const uint32_t lenx = (x1 >> (s1 - ext)) & ~(0xffffffffu << ext);
        const uint32_t distx = (x2 >> (s2 - dext)) & ~(0xffffffffu << dext);
        x1 = x1n;
        const bool emit = act && sym != 256u;
        if (emit && lane == j) {
          ta[r] = sym | (lenx << 9) | (e2 << 14);
          tb[r] = distx | (((b.wi << 5) | b.bo) << 13);  // + low bits of the reader position after the token
        }
        ntok += emit ? 1u : 0u;
        act = emit && !b.overrun;
      }
    }
    uint32_t bad_k = 0, bad_back = 0;
    // only the counting and the marker kernels ever see a segment with a window in front of it (and the byte
    // kernel's dictionary instantiation, a member with its dictionary window in front)
    const uint32_t win = (COUNT_ONLY || sizeof(OutT) == 2 || DICT) ? g.win : 0u;
    const int fev = flush_tokens<COUNT_ONLY, OutT, DICT>(g.out, op, g.cap, win, ta, tb, ntok, len_addr, dist_addr, bad_k,
                                                          bad_back, wend);
    // a group that stopped: end of block (symbol 256), or a reader far past the end of its input
    ev = (act0 && !act) ? (b.overrun ? 100 + ZB_ERR_END_OF_BUFFER : 1) : 0;
    if (fev) {
      // inflate.nim:190-225 order: a token that ran off the input reports the end of the buffer, but a
      // length symbol >= 29 or a distance symbol >= 30 is invalid wherever the input ends, as long as the
      // literal/length code itself was read in full: for those, the end is checked where that code ends
      // (a length symbol >= 29 has no distance after it in the token; bad_back covers the distance case)
      uint32_t pk = 0;
#pragma unroll
      for (int r = 0; r < INF_ROUNDS; r++) {
        const uint32_t v = g_shfl(tb[r], (int)(bad_k & (uint32_t)(INF_G - 1)));
        if ((bad_k / (uint32_t)INF_G) == (uint32_t)r) pk = v >> 13;
      }
      pk -= bad_back;
      const uint64_t now_abs = br_consumed_abs(b);  // the token lies < 2^11 bits before this
      const bool past = now_abs - (uint64_t)(((uint32_t)now_abs - pk) & 0x7ffffu) > b.end_bit;
      ev = 100 + (past ? ZB_ERR_END_OF_BUFFER : (fev == 2 ? ZB_ERR_UNCOMPRESS : ZB_ERR_DST_TOO_SMALL));
    }
    if (__any_sync(FULL_MASK, ev != 0)) break;
  }
  g.op = op;
  return ev;
}

#ifndef INF_MIN_CTAS
#define INF_MIN_CTAS 5   // register budget for 5 CTAs (20 warps) per SM, the shared-memory limit
#endif
// DICT: whole members decoded against their dictionaries (ZbInflateWork::mdict); <true, false, true> counts,
// <false, false, true> writes bytes.  The instantiations without it compile as they did before the dictionary existed.
template <bool COUNT_ONLY, bool MARK, bool DICT = false>
__global__ void __launch_bounds__(INF_THREADS, INF_MIN_CTAS)
    k_inflate(ZbInflateWork w) {
  typedef typename std::conditional<MARK, uint16_t, uint8_t>::type OutT;
  extern __shared__ __align__(16) unsigned char inf_smem[];
  // base | extra bits << 16 (RFC 1951 3.2.5), unused slots 0; placed after the groups' tables
  uint32_t *len_tab = reinterpret_cast<uint32_t *>(inf_smem + INF_GROUPS * sizeof(GroupSmem));
  uint32_t *dist_tab = len_tab + 32;
  const uint32_t tab_addr = (uint32_t)__cvta_generic_to_shared(len_tab);
  const int lane = g_lane();
  GroupSmem *gs = reinterpret_cast<GroupSmem *>(inf_smem) + threadIdx.x / INF_G;
  if (threadIdx.x < 32)
    len_tab[threadIdx.x] = threadIdx.x < 29 ? (zb_len_base((int)threadIdx.x) | ((uint32_t)zb_len_extra_bits((int)threadIdx.x) << 16)) : 0u;
  else if (threadIdx.x < 64) {
    int c = (int)threadIdx.x - 32;
    dist_tab[c] = c < 30 ? (zb_dist_base(c) | ((uint32_t)zb_dist_extra_bits(c) << 16)) : 0u;
  }
  __syncthreads();
  Grp<OutT> g;
  g.st = ST_FETCH;
  g.win = 0;
  g.gate = 0;
  g.ready_seen = 0;
  g.b.gbase = nullptr;
  g.b.nwords = 0;
  g.b.last_mask = 0;
  g.b.cur = g.b.nxt = 0;
  g.b.w0 = g.b.w1 = g.b.w2 = g.b.wi = g.b.bo = 0;
  g.b.end_bit = 0;
  g.b.overrun = false;
  g.op = g.cap = 0;
  g.out = nullptr;
  uint32_t rec_k = 0;   // the recorder's next multiple of 32768 (counting instantiation only)
  const uint8_t *wend = nullptr;  // DICT: just past the current member's W
  for (;;) {
    int done = 1;  // status to report when `fin` is set
    bool fin = false;
    if (g.st == ST_FETCH) {
      uint32_t i = 0;
      if (lane == 0) i = atomicAdd(w.counter, 1u);
      i = g_shfl(i, 0);
      if (i < w.n && w.gate_first) {
        // the member's input may still be on its way: wait for its copy-in group (lane 0 polls, the group follows)
        uint32_t gt = 0;
        while (gt + 1u < w.n_gates && i >= w.gate_first[gt + 1u]) gt++;
        g.gate = gt;
        if (gt >= g.ready_seen) {
          // (an acquire load also drops this SM's L1 lines: a line read before the copy-in landed may hold stale
          // bytes of this member's head.  The count only grows, so a group asks once per copy-in group.)
          uint32_t r = 0;
          if (lane == 0) {
            r = gate_load(w.gate_ready);
            if (r <= gt) {
              const uint64_t t0 = gate_clock();
              while ((r = gate_load(w.gate_ready)) <= gt && gate_clock() - t0 < 30000000000ull) __nanosleep(500);
            }
          }
          g.ready_seen = g_shfl(r, 0);
        }
      }
      if (i < w.n && w.order) i = w.order[i];
      if (i >= w.n) {
        g.st = ST_EXIT;
      } else if (w.skip && w.skip[i]) {
        // handled elsewhere (a large member decoded as parallel segments): fetch the next one
        gate_member_done(w, g.gate);
      } else if ((COUNT_ONLY || MARK) && w.seg_bits) {
        // a speculative segment of one raw stream: bit-exact start and end inside w.src; bits beyond the
        // end are the next segment's (real data), so an over-read is harmless and an over-RUN is caught
        const uint64_t sb = w.seg_bits[2 * i], eb = w.seg_bits[2 * i + 1];
        const uint64_t byte0 = sb >> 3;
        g.idx = i;
        g.src = w.src + byte0;
        g.len = w.seg_limit - byte0;
        g.op = 0;
        g.final_block = false;
        g.kind = ZB_DF_DEFLATE;
        g.expect = 0;
        g.win = (i == 0 && !w.seg_win0) ? 0u : 32768u;   // segment 0 starts the stream: it has no window
        g.out = COUNT_ONLY ? nullptr : reinterpret_cast<OutT *>(w.dst) + w.dst_off[i];
        const uint64_t cap64 = COUNT_ONLY ? ~0ull : w.dst_off[i + 1] - w.dst_off[i];
        g.cap = (uint32_t)min(cap64, (uint64_t)0xfffffdffu - 32768u);
        g.shift0 = (uint32_t)((uintptr_t)g.src & 3u);
        g.b.gbase = reinterpret_cast<const uint32_t *>(g.src - g.shift0);
        g.b.nwords = (uint32_t)min((uint64_t)0xffffffffu, (g.shift0 + g.len + 3u) >> 2);
        g.b.last_mask = ((g.shift0 + g.len + 3u) >> 2) > 0xffffffffull ? 0xffffffffu : br_tail_mask(g.shift0 + g.len);
        g.b.end_bit = g.shift0 * 8ull + (eb - byte0 * 8ull);
        g.b.overrun = false;
        br_seek(g.b, g.shift0, 0);
        br_skip<false>(g.b, (uint32_t)(sb & 7ull));
        if (COUNT_ONLY && w.rec) rec_k = i == 0 ? 0u : (uint32_t)(w.rec_base[i] / 32768ull + 1ull);
        g.st = ST_BLOCK;
      } else {
        const uint64_t s0 = w.src_off[i], s1 = w.src_off[i + 1];
        g.idx = i;
        g.win = 0;
        g.src = w.src + s0;
        g.len = s1 - s0;
        g.op = 0;
        g.final_block = false;
        uint64_t pos = 0;
        uint32_t isize = 0;
        g.kind = 0;
        g.expect = 0;
        int st;
        if (DICT) {
          // a member without a dictionary parses as in the plain instantiation: FDICT is ZB_ERR_FDICT
          const ZbMemberDict md = w.mdict[i];
          st = zb_parse_wrapper(g.src, g.len, w.data_format, w.pos, pos, g.kind, g.expect, isize,
                                md.win_len ? &md.dict_id : nullptr);
          // raw members, and zlib members whose FDICT was accepted (payload at 6), see the window
          g.win = (g.kind == ZB_DF_DEFLATE || (g.kind == ZB_DF_ZLIB && pos == 6)) ? md.win_len : 0u;
          wend = md.wend;
        } else {
          st = zb_parse_wrapper(g.src, g.len, w.data_format, w.pos, pos, g.kind, g.expect, isize);
        }
        if (st == ZB_OK && COUNT_ONLY && g.kind == ZB_DF_GZIP) {
          g.op = isize;  // gzip.nim:66 (trustSize's source)
          fin = true;
          done = ZB_OK;
        } else if (st != ZB_OK) {
          fin = true;
          done = st;
        } else {
          g.out = COUNT_ONLY ? nullptr : reinterpret_cast<OutT *>(w.dst) + w.dst_off[i];
          const uint64_t cap64 = COUNT_ONLY ? ~0ull : w.dst_off[i + 1] - w.dst_off[i];
          // positions are 32-bit inside a member (a single member's output is limited to 4 GiB - 1);
          // op + tlen is computed in 32 bits: keep 512 bytes of headroom below 2^32
          g.cap = (uint32_t)min(cap64, (uint64_t)0xfffffdffu);
          g.shift0 = (uint32_t)((uintptr_t)g.src & 3u);
          g.b.gbase = reinterpret_cast<const uint32_t *>(g.src - g.shift0);
          g.b.nwords = (uint32_t)((g.shift0 + g.len + 3u) >> 2);
          g.b.last_mask = br_tail_mask(g.shift0 + g.len);
          g.b.end_bit = (g.shift0 + g.len) * 8ull;
          g.b.overrun = false;
          br_seek(g.b, g.shift0, pos);
          g.st = ST_BLOCK;
        }
      }
    } else if (g.st == ST_BLOCK && w.seg_mode && br_consumed_abs(g.b) == g.b.end_bit) {
      fin = true;  // the segment's input is used up at a block boundary
      done = ZB_OK;
    } else if (g.st == ST_BLOCK) {
      if (COUNT_ONLY && w.resume && g.idx + 1u == w.n && lane == 0) {
        // the open segment of a decompress stream: where it resumes if this block does not complete.  (A segment
        // whose input is used up at a block boundary ends in the branch above, with status ZB_OK: it resumes there.
        // The marker pass decodes that segment again as a closed one, up to the block boundary found here.)
        w.resume[0] = (uint64_t)(reinterpret_cast<const uint8_t *>(g.b.gbase) - w.src) * 8ull + br_consumed_abs(g.b);
        w.resume[1] = g.op;
      }
      if (COUNT_ONLY && w.rec && lane == 0) {
        // an access point for every multiple of 32768 this block start is the first one at or past
        const uint64_t o = w.rec_base[g.idx] + g.op;
        if (rec_k < w.nrec && (uint64_t)rec_k * 32768ull <= o) {
          const uint64_t bit = (uint64_t)(reinterpret_cast<const uint8_t *>(g.b.gbase) - w.src) * 8ull + br_consumed_abs(g.b);
          do {
            w.rec[2 * rec_k] = bit;
            w.rec[2 * rec_k + 1] = o;
            rec_k++;
          } while (rec_k < w.nrec && (uint64_t)rec_k * 32768ull <= o);
        }
      }
      int r = begin_block<COUNT_ONLY, OutT>(g, gs);
      if (r >= 0) {
        fin = true;
        done = r;
      } else if (r == BLK_SYMS) {
        g.st = ST_SYMS;
      } else if (g.final_block) {
        fin = true;
        done = ZB_OK;
      }
    }
    if (fin) {
      if (lane == 0) {
        w.status[g.idx] = done;
        w.out_len[g.idx] = done == ZB_OK ? (uint64_t)g.op : 0ull;
        w.kind[g.idx] = w.seg_mode ? (uint32_t)g.final_block : g.kind;
        w.expect[g.idx] = g.expect;
      }
      gate_member_done(w, g.gate);
      g.st = ST_FETCH;
    }
    __syncwarp();
    if (__all_sync(FULL_MASK, g.st == ST_EXIT)) break;
    // run the lockstep symbol loop only when no group of the warp is waiting for a header or a
    // new member: those are short, and would otherwise stall behind a whole block of symbols
    if (__any_sync(FULL_MASK, g.st == ST_FETCH || g.st == ST_BLOCK)) continue;
    const int ev = symbol_loop<COUNT_ONLY, OutT, DICT>(g, gs, tab_addr, wend);
    if (g.st == ST_SYMS && ev) {
      int st = ZB_OK;
      if (ev == 1) {
        if (br_past_end(g.b)) st = ZB_ERR_END_OF_BUFFER;
      } else {
        st = ev - 100;
      }
      if (st != ZB_OK || g.final_block) {
        if (lane == 0) {
          w.status[g.idx] = st;
          w.out_len[g.idx] = st == ZB_OK ? (uint64_t)g.op : 0ull;
          w.kind[g.idx] = w.seg_mode ? (uint32_t)g.final_block : g.kind;
          w.expect[g.idx] = g.expect;
        }
        gate_member_done(w, g.gate);
        g.st = ST_FETCH;
      } else {
        g.st = ST_BLOCK;
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// Blocked combine-reduce checksums (replaces crc32 crc.nim:53 / crc32_simd.nim:39-144 and
// adler32 adler32.nim:6 / adler32_simd.nim:45-120, and the trailer checks gzip.nim:80-88,
// zippy.nim:154-162).  A buffer is cut into 64 KiB pieces; k_piece_checksum gives every piece
// to one CTA (TMA-staged, 8 warps x 8 KiB, lane-strided CRC stepping + dp4a Adler sums, see
// zb_device.cuh), k_buffer_combine folds a buffer's pieces with x^(8*len) multiplications /
// the closed-form Adler merge, and in verify mode compares with the trailer.
#define CK_PIECE ZB_CK_PIECE_BYTES
#define CK_THREADS 512
#define CK_WARPS (CK_THREADS / 32)
#define CK_WARP_BYTES (CK_PIECE / CK_WARPS)          // 2 KiB per warp and piece (Adler, ragged pieces)
#define CK_ROWS (CK_PIECE / 128)                      // a full piece is 256 rows of 128 B
#define CK_CHAINS (CK_WARPS * 4)                      // CRC of a full piece: row q + 64 k belongs to chain q, warp w owns chains w + 16 c
#define CK_PARTIAL_WORDS (CK_WARPS * 32)              // what the CRC path leaves per full piece: one word per warp and lane
#define CK_STAGES 2
#define CK_STAGE_BYTES (CK_PIECE + 128)
#define CK_SM_REP (CK_STAGES * CK_STAGE_BYTES)        // chain step tables (x^(8*128*64)), one copy per lane (bank): 4 x 256 x 32 words
#define CK_SM_T1024 (CK_SM_REP + 4 * 256 * 32 * 4)    // x^1024 step table (ragged pieces)
#define CK_SM_QT (CK_SM_T1024 + 4 * 256 * 4)          // chain join tables: multiply by x^(8*128*16*k), k = 1..3
#define CK_SM_LMUL (CK_SM_QT + 3 * 4 * 256 * 4)
#define CK_LMUL_WORDS 52
#define CK_SM_PART (CK_SM_LMUL + CK_LMUL_WORDS * 4)
#define CK_SM_BAR (CK_SM_PART + CK_WARPS * 24)
#define CK_SM_TOTAL (CK_SM_BAR + 16 * CK_STAGES + 8)
static_assert(CK_SM_TOTAL <= 232448, "one CTA per SM");
static_assert(CK_ROWS == 4 * CK_CHAINS, "four rows per chain");
static_assert(CK_PARTIAL_WORDS * 4 == ZB_CK_PARTIAL_BYTES, "scratch size");

__device__ __forceinline__ uint32_t piece_len(uint64_t buflen, uint64_t rel) {
  return rel < buflen ? (uint32_t)min((uint64_t)CK_PIECE, buflen - rel) : 0u;
}
__device__ __forceinline__ uint32_t ck_piece_info(const ZbChecksumWork &w, uint32_t pid, const uint8_t *&src, uint32_t &kind) {
  const ZbPiece pc = w.pieces[pid];
  uint64_t buflen = w.lens ? w.lens[pc.buf] : w.off[pc.buf + 1] - w.off[pc.buf];
  if (w.status && w.status[pc.buf] != ZB_OK) buflen = 0;
  kind = (uint32_t)w.kind;
  if (w.kinds) {
    const uint32_t kd = w.kinds[pc.buf];
    kind = kd == ZB_DF_ZLIB ? 1u : 0u;
    if (kd != ZB_DF_GZIP && kd != ZB_DF_ZLIB) buflen = 0;   // raw deflate: nothing to verify
  }
  src = w.src + w.off[pc.buf] + pc.rel;
  return piece_len(buflen, pc.rel);
}

// multiply by the chain step with the lane's own copy of the tables: entry (j, b) of lane l at
// rep[((j * 256 + b) * 32) + l], i.e. always in bank l -- four conflict-free lookups (a shared 4 KiB table
// cost ~3.5 wavefronts per lookup)
__device__ __forceinline__ uint32_t ck_mul_rep(const uint32_t *rep_lane, uint32_t r) {
  return rep_lane[(r & 255u) * 32u] ^ rep_lane[(256u + ((r >> 8) & 255u)) * 32u] ^ rep_lane[(512u + ((r >> 16) & 255u)) * 32u] ^
         rep_lane[(768u + (r >> 24)) * 32u];
}
__device__ __forceinline__ uint32_t ck_mul_tab(const uint32_t *t /*[4][256]*/, uint32_t r) {
  return t[r & 255u] ^ t[256 + ((r >> 8) & 255u)] ^ t[512 + ((r >> 16) & 255u)] ^ t[768 + (r >> 24)];
}

// CRC-32 of a FULL staged piece, this warp's share: lane i takes word i of the rows of four chains (row q + 64 k,
// q = warp + 16 c), Horner inside a chain with the 64-row step, then the four chains are joined with table
// multiplications.  What is left per warp and lane is one word whose weight is x^(1024 * (15 - warp)) * x^(32 * (31 -
// lane)): the 16 x 32 words of a piece are a 2 KiB message with the piece's raw CRC, folded by k_piece_fold -- no
// generic GF(2) multiplication and no cross-warp exchange here (both together were over a third of this kernel's instructions).
template <bool ALIGNED>
__device__ __forceinline__ uint32_t ck_warp_crc_rows(const uint8_t *data, uint32_t mis, int warp, const uint32_t *rep_lane,
                                                     const uint32_t *jt) {
  const uint32_t o = mis + 4u * (uint32_t)zb_lane() + 128u * (uint32_t)warp;
  uint32_t r[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (uint32_t k = 0; k < CK_ROWS / CK_CHAINS; k++) {
    uint32_t wv[4];
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
      const uint32_t off = o + 128u * (CK_CHAINS * k + CK_WARPS * c);
      wv[c] = ALIGNED ? *reinterpret_cast<const uint32_t *>(data + off) : zb_ld32_unaligned(data, off);
    }
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
      if (k) r[c] = ck_mul_rep(rep_lane, r[c]);
      r[c] ^= wv[c];
    }
  }
  return ck_mul_tab(jt + 2 * 1024, r[0]) ^ ck_mul_tab(jt + 1024, r[1]) ^ ck_mul_tab(jt, r[2]) ^ r[3];
}

// Adler sums of one warp's WB bytes (2 or 4 KiB) of a staged piece: lane i takes word i of every 128-byte row, four
// rows per step.
template <uint32_t WB>
__device__ __forceinline__ ZbCheck ck_warp_adler(const uint8_t *base, uint32_t off) {
  const int lane = zb_lane();
  constexpr uint32_t QR = WB / 512;   // steps
  constexpr uint32_t QB = WB / 4;     // bytes per quarter
  const uint32_t o = off + 4u * (uint32_t)lane, rel0 = 4u * (uint32_t)lane;
  uint32_t a = 0;
  uint64_t b = 0;
#pragma unroll 2
  for (uint32_t k = 0; k < QR; k++) {
    const uint32_t w0 = zb_ld32_unaligned(base, o + 128u * k), w1 = zb_ld32_unaligned(base, o + 128u * (QR + k));
    const uint32_t w2 = zb_ld32_unaligned(base, o + 128u * (2u * QR + k)), w3 = zb_ld32_unaligned(base, o + 128u * (3u * QR + k));
    const uint32_t s0 = __dp4a(w0, 0x01010101u, 0u), s1 = __dp4a(w1, 0x01010101u, 0u);
    const uint32_t s2 = __dp4a(w2, 0x01010101u, 0u), s3 = __dp4a(w3, 0x01010101u, 0u);
    a += s0 + s1 + s2 + s3;
    const uint32_t rel = rel0 + 128u * k;
    // (WB - position) * byte sums fit in 32 bits per row: 4096 * 4 * 1020 < 2^32
    b += (uint64_t)((4u * QB - rel) * s0 + (3u * QB - rel) * s1) + (uint64_t)((2u * QB - rel) * s2 + (QB - rel) * s3);
    b -= (uint64_t)(__dp4a(w0, 0x03020100u, 0u) + __dp4a(w1, 0x03020100u, 0u) + __dp4a(w2, 0x03020100u, 0u) +
                    __dp4a(w3, 0x03020100u, 0u));
  }
  ZbCheck out;
  out.crc_raw = 0;
  out.a_sum = zb_warp_sum64((uint64_t)a);
  out.b_sum = zb_warp_sum64(b);
  return out;
}

// Adler sums of a ragged piece of n bytes (no tables): lane-strided words, the last 1..3 bytes by lane 0
__device__ __forceinline__ ZbCheck ck_warp_adler_ragged(const uint8_t *base, uint32_t off, uint32_t n) {
  const int lane = zb_lane();
  uint64_t a = 0, b = 0;
  for (uint32_t i = 4u * (uint32_t)lane; i + 4u <= n; i += 128u) {
    const uint32_t w = zb_ld32_unaligned(base, off + i);
    const uint32_t s = __dp4a(w, 0x01010101u, 0u);
    a += s;
    b += (uint64_t)(n - i) * s - __dp4a(w, 0x03020100u, 0u);
  }
  if (lane == 0)
    for (uint32_t i = n & ~3u; i < n; i++) {
      a += base[off + i];
      b += (uint64_t)(n - i) * base[off + i];
    }
  ZbCheck out;
  out.crc_raw = 0;
  out.a_sum = zb_warp_sum64(a);
  out.b_sum = zb_warp_sum64(b);
  return out;
}

// Persistent CTAs, a ring of 32 KiB shared-memory stages filled by TMA bulk copies: while the 16 warps checksum
// stage k, the copy for k+1 is in flight.  Piece descriptors (source pointer, length, kind: dependent global
// loads) are fetched 16..32 pieces ahead into a small shared ring so they never sit on the critical path.
// CRC-32 and Adler-32 are separate paths (a piece needs one of them): Adler is two dp4a per word and runs at the
// copy rate; CRC-32 without a carry-less multiply is one table lookup per byte, which is why the step tables are
// replicated per bank (one CTA per SM).  A full CRC piece leaves 16 x 32 partial words (ck_warp_crc_rows) in
// w.partials for k_piece_fold; every other piece (Adler, ragged, empty) gets its piece_out entry here.
// ADLER_ONLY: every piece wants Adler-32 (the adler32 entry points): no CRC tables in shared memory, so three
// CTAs share an SM and three times as many bulk copies are in flight.
#define CK_SM_TOTAL_ADLER (CK_SM_REP + CK_LMUL_WORDS * 4 + CK_WARPS * 24 + 16 * CK_STAGES + 8)
#define CK_INFO 32
#define CK_THREADS_ADLER 256   // the Adler-only CTAs: 8 warps x 4 KiB (three CTAs per SM)
template <bool ADLER_ONLY>
__global__ void __launch_bounds__(ADLER_ONLY ? CK_THREADS_ADLER : CK_THREADS, ADLER_ONLY ? 3 : 1)
    k_piece_checksum(ZbChecksumWork w) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int NT = ADLER_ONLY ? CK_THREADS_ADLER : CK_THREADS, NW = NT / 32;
  constexpr uint32_t WB = CK_PIECE / NW;   // bytes per warp and piece on the Adler / ragged paths
  constexpr uint32_t LMUL_OFF = ADLER_ONLY ? CK_SM_REP : CK_SM_LMUL;
  uint32_t *rep = reinterpret_cast<uint32_t *>(smem + CK_SM_REP);
  uint32_t *t1024 = reinterpret_cast<uint32_t *>(smem + CK_SM_T1024);
  uint32_t *qt = reinterpret_cast<uint32_t *>(smem + CK_SM_QT);
  uint32_t *lane_mul = reinterpret_cast<uint32_t *>(smem + LMUL_OFF);
  uint64_t *part = reinterpret_cast<uint64_t *>(smem + LMUL_OFF + CK_LMUL_WORDS * 4);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + LMUL_OFF + CK_LMUL_WORDS * 4 + CK_WARPS * 24);
  __shared__ const uint8_t *info_src[CK_INFO];
  __shared__ uint32_t info_len[CK_INFO];
  __shared__ uint32_t info_kind[CK_INFO];
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t stride = gridDim.x;
  if (tid == 0) {
    for (int i = 0; i < CK_STAGES; i++) {
      zb_mbar_init(&bars[i], 1);
      zb_mbar_init(&bars[CK_STAGES + i], NW);   // "stage i has been read by every warp" (full CRC pieces)
    }
    zb_fence_mbar_init();
  }
  if (!ADLER_ONLY) {
    const uint32_t *t = &w.tabs->mul64r[0][0];
    for (int i = tid; i < 1024 * 32; i += NT) rep[i] = t[i >> 5];   // entry e, lane l at rep[e * 32 + l]
    const uint32_t *t1 = &w.tabs->mul1024[0][0];
    for (int i = tid; i < 1024; i += NT) t1024[i] = t1[i];
    const uint32_t *q = &w.tabs->ck_join[0][0][0];
    for (int i = tid; i < 3 * 1024; i += NT) qt[i] = q[i];
    if (tid < 33) lane_mul[tid] = w.tabs->lane_mul[tid];
    if (tid >= 64 && tid < 80) lane_mul[33 + tid - 64] = w.tabs->ck_sub[tid - 64];
  }
  if (tid >= 128 && tid < 128 + CK_INFO) {  // descriptors of this CTA's first 32 pieces
    const uint32_t j = (uint32_t)tid - 128u, pid = blockIdx.x + j * stride;
    const uint8_t *src = nullptr;
    uint32_t kd = 0;
    info_len[j] = pid < w.n_pieces ? ck_piece_info(w, pid, src, kd) : 0u;
    info_src[j] = src;
    info_kind[j] = kd;
  }
  __syncthreads();
  if (tid == 0) {  // prologue: fill the ring
    for (uint32_t k = 0; k < CK_STAGES; k++) {
      if (blockIdx.x + k * stride >= w.n_pieces) break;
      if (info_len[k]) zb_stage_chunk(smem + k * CK_STAGE_BYTES, info_src[k], info_len[k], &bars[k]);
    }
  }
  const uint32_t *rep_lane = rep + lane;
  uint32_t k = 0, phases = 0;  // bit s of `phases` = parity of the next completion of stage s
  uint32_t ephases = 0;        // the same for the stages' "read by every warp" barriers
  for (uint32_t pid = blockIdx.x; pid < w.n_pieces; pid += stride, k++) {
    const uint32_t stage = k % CK_STAGES;
    const uint32_t len = info_len[k % CK_INFO], kind = info_kind[k % CK_INFO];
    const uint8_t *src = info_src[k % CK_INFO];
    const uint8_t *data = smem + stage * CK_STAGE_BYTES;
    const uint32_t mis = (uint32_t)((uintptr_t)src & 15u);
    if (len) {  // empty pieces are never copied, so their stage's phase does not advance
      zb_mbar_wait(&bars[stage], (phases >> stage) & 1u);
      phases ^= 1u << stage;
    }
    const bool full_crc = !ADLER_ONLY && len == CK_PIECE && kind == 0u;
    if (full_crc) {
      const uint32_t r = (mis & 3u) ? ck_warp_crc_rows<false>(data, mis, warp, rep_lane, qt) : ck_warp_crc_rows<true>(data, mis, warp, rep_lane, qt);
      w.partials[(size_t)pid * CK_PARTIAL_WORDS + (uint32_t)tid] = r;
    } else {
      const uint32_t b0 = (uint32_t)warp * WB, b1 = min(b0 + WB, len);
      ZbCheck c;
      c.crc_raw = 0;
      c.a_sum = c.b_sum = 0;
      if (b0 < len) {
        const uint32_t n = b1 - b0;
        if (ADLER_ONLY || kind) c = n == WB ? ck_warp_adler<WB>(data, mis + b0) : ck_warp_adler_ragged(data, mis + b0, n);
        else c = zb_warp_checksums(data, mis + b0, n, t1024, lane_mul);   // a buffer's ragged last piece
        const uint32_t after = len - b1;
        if (after) {
          if (!ADLER_ONLY && kind == 0)
            c.crc_raw = zb_gf2_mul(c.crc_raw, (after & (CK_WARP_BYTES - 1u)) == 0u ? lane_mul[33 + after / CK_WARP_BYTES] : zb_xpow8_t(w.tabs->pow2, after));
          else c.b_sum += (uint64_t)after * c.a_sum;
        }
      }
      if (lane == 0) {
        part[warp * 3 + 0] = c.crc_raw;
        part[warp * 3 + 1] = c.a_sum;
        part[warp * 3 + 2] = c.b_sum;
      }
    }
    // every warp is done with this stage (and with info slot k) before it is refilled.  After a full CRC piece only
    // thread 0 has to know: the warps signal an mbarrier and run on into the other stage
    if (full_crc && (k % 16u) != 15u) {
      __syncwarp();
      if (lane == 0) zb_mbar_arrive(&bars[CK_STAGES + stage]);
      if (tid == 0) zb_mbar_wait(&bars[CK_STAGES + stage], (ephases >> stage) & 1u);
      ephases ^= 1u << stage;
    } else {
      __syncthreads();
    }
    if (tid == 0) {
      // refill this stage with the piece CK_STAGES iterations ahead
      const uint32_t nk = k + CK_STAGES;
      if (pid + CK_STAGES * stride < w.n_pieces && info_len[nk % CK_INFO])
        zb_stage_chunk(smem + stage * CK_STAGE_BYTES, info_src[nk % CK_INFO], info_len[nk % CK_INFO], &bars[stage]);
      if (!full_crc) {
        uint32_t raw = 0;
        uint64_t a = 0, b = 0;
        for (int j = 0; j < NW; j++) {
          raw ^= (uint32_t)part[j * 3 + 0];
          a += part[j * 3 + 1];
          b += part[j * 3 + 2];
        }
        ZbChunkCheck cc;
        cc.crc_raw = raw;
        cc.adler = ((uint32_t)(b % ZB_ADLER_MOD) << 16) | (uint32_t)(a % ZB_ADLER_MOD);  // (B mod p, A mod p), not yet an Adler value
        w.piece_out[pid] = cc;
      }
    } else if (warp == 1 && (k % 16u) == 15u && lane < 16) {
      // descriptors for pieces k+17 .. k+32 go into the half of the ring that has just been used up
      const uint32_t j = k + 17u + (uint32_t)lane, npid = blockIdx.x + j * stride;
      const uint8_t *nsrc = nullptr;
      uint32_t kd = 0;
      info_len[j % CK_INFO] = npid < w.n_pieces ? ck_piece_info(w, npid, nsrc, kd) : 0u;
      info_src[j % CK_INFO] = nsrc;
      info_kind[j % CK_INFO] = kd;
    }
    // part[] and the descriptor ring are consistent for the next piece.  A full CRC piece touches neither (its words
    // went to w.partials), so between descriptor refreshes the warps may run on into the next stage.
    if (!full_crc || (k % 16u) == 15u) __syncthreads();
  }
}

// Second step of the CRC path: one warp per full piece folds its 16 x 32 partial words -- a 2 KiB message in the
// usual lane-strided layout -- into the piece's raw CRC: 15 steps of x^1024, ONE generic GF(2) multiplication
// per lane for the lane shifts, a warp XOR.  (6 % of the bytes of the first step, and as parallel as it.)
__global__ void __launch_bounds__(256)
    k_piece_fold(ZbChecksumWork w) {
  __shared__ uint32_t tab[1024];
  __shared__ uint32_t lmul[33];
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 1024; i += 256) tab[i] = (&w.tabs->mul1024[0][0])[i];
  if (tid < 33) lmul[tid] = w.tabs->lane_mul[tid];
  __syncthreads();
  for (uint32_t pid = blockIdx.x * 8u + (uint32_t)warp; pid < w.n_pieces; pid += gridDim.x * 8u) {
    const uint8_t *src = nullptr;
    uint32_t kind = 0;
    const uint32_t len = ck_piece_info(w, pid, src, kind);
    if (len != CK_PIECE || kind != 0u) continue;  // k_piece_checksum wrote this piece's entry itself
    const uint32_t *m = w.partials + (size_t)pid * CK_PARTIAL_WORDS + (uint32_t)lane;
    uint32_t v[CK_WARPS];
#pragma unroll
    for (uint32_t row = 0; row < CK_WARPS; row++) v[row] = __ldcs(m + row * 32u);
    uint32_t r = v[0];
#pragma unroll
    for (uint32_t row = 1; row < CK_WARPS; row++) r = zb_mul1024(tab, r) ^ v[row];
    r = zb_warp_xor(zb_gf2_mul(r, lmul[32 - lane]));
    if (lane == 0) {
      ZbChunkCheck cc;
      cc.crc_raw = r;
      cc.adler = 0;
      w.piece_out[pid] = cc;
    }
  }
}

// raw CRC (init 0) / Adler sums of a whole buffer -> the checksum value; store and, in verify mode, compare
__device__ __forceinline__ void ck_finish(const ZbChecksumWork &w, uint32_t i, int kind, uint32_t r, uint64_t a, uint64_t b,
                                          uint64_t buflen) {
  const uint32_t v = kind == 0 ? ~(zb_gf2_mul(buflen == ZB_CHUNK_BYTES ? w.tabs->sub_mul[0] : zb_xpow8_t(w.tabs->pow2, buflen), 0xffffffffu) ^ r)
                               : zb_adler_from_sums(a % ZB_ADLER_MOD, b % ZB_ADLER_MOD, buflen);
  if (w.out) w.out[i] = v;
  if (w.expect) {
    if (v != w.expect[i]) w.status[i] = ZB_ERR_CHECKSUM;
    else if (kind == 0 && w.isize_src) {
      const uint8_t *t = w.isize_src + w.isize_off[i + 1] - 4;
      if (zb_ld_le32(t) != (uint32_t)buflen) w.status[i] = ZB_ERR_SIZE;
    }
  }
}

// One warp per buffer: lane j folds pieces j, j+32, ... (Horner in x^(8 * 32 * 64 KiB)), the lane
// results are shifted to the end of the buffer and XOR-reduced; Adler sums add up directly.
__global__ void __launch_bounds__(128)
    k_buffer_combine(ZbChecksumWork w) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = (int)(threadIdx.x & 31u);
  if (i >= w.n) return;
  if (w.status && w.status[i] != ZB_OK) return;
  int kind = w.kind;
  if (w.kinds) {
    const uint32_t kd = w.kinds[i];
    if (kd == ZB_DF_GZIP) kind = 0;
    else if (kd == ZB_DF_ZLIB) kind = 1;
    else return;  // raw deflate: nothing to verify
  }
  const uint64_t buflen = w.lens ? w.lens[i] : w.off[i + 1] - w.off[i];
  const uint32_t p0 = w.first[i];
  const uint32_t np = (uint32_t)((buflen + CK_PIECE - 1) / CK_PIECE);  // pieces that hold data
  if (w.big_pieces && np > w.big_pieces) return;  // k_buffer_combine_big's
  uint32_t r = 0;
  uint64_t a = 0, b = 0, end = 0;  // end = bytes from the buffer start to the end of this lane's last piece
  if (kind == 0) {
    uint32_t step = 0;  // x^(8 * 32 * 64 KiB), computed only if a lane has more than one piece
    for (uint32_t k = (uint32_t)lane; k < np; k += 32) {
      const uint32_t l = piece_len(buflen, (uint64_t)k * CK_PIECE);
      const uint32_t raw = w.piece_out[p0 + k].crc_raw;
      if (k >= 32) {
        if (l == CK_PIECE) {
          if (!step) step = zb_xpow8_t(w.tabs->pow2, 32ull * CK_PIECE);
          r = zb_gf2_mul(r, step);
        } else {
          r = zb_gf2_mul(r, zb_xpow8_t(w.tabs->pow2, 31ull * CK_PIECE + l));
        }
      }
      r ^= raw;
      end = (uint64_t)k * CK_PIECE + l;
    }
    if ((uint32_t)lane < np && end < buflen) r = zb_gf2_mul(r, zb_xpow8_t(w.tabs->pow2, buflen - end));
    r = zb_warp_xor(r);
  } else {
    for (uint32_t k = (uint32_t)lane; k < np; k += 32) {
      const uint32_t l = piece_len(buflen, (uint64_t)k * CK_PIECE);
      const uint32_t ab = w.piece_out[p0 + k].adler;
      const uint64_t ak = ab & 0xffffu, bk = ab >> 16;
      const uint64_t after = (buflen - ((uint64_t)k * CK_PIECE + l)) % ZB_ADLER_MOD;
      a += ak;
      b = (b + bk + after * ak) % ZB_ADLER_MOD;
    }
    a = zb_warp_sum64(a % ZB_ADLER_MOD);
    b = zb_warp_sum64(b);
  }
  if (lane != 0) return;
  ck_finish(w, i, kind, r, a, b, buflen);
}

// The same fold for a buffer of very many pieces (one multi-GiB input of crc32 / adler32): 1024 threads, thread t
// folds pieces t, t + 1024, ... (Horner in x^(8 * 1024 * 32 KiB)), shifts to the end of the buffer, block XOR / sum.
// (One warp per buffer took longer to fold the 131072 pieces of a 4 GiB buffer than the pieces took.)
#define CKB_THREADS 1024
__global__ void __launch_bounds__(CKB_THREADS)
    k_buffer_combine_big(ZbChecksumWork w) {
  const uint32_t i = blockIdx.x;
  __shared__ uint32_t red_r[CKB_THREADS / 32];
  __shared__ uint64_t red_a[CKB_THREADS / 32], red_b[CKB_THREADS / 32];
  if (w.status && w.status[i] != ZB_OK) return;
  int kind = w.kind;
  if (w.kinds) {
    const uint32_t kd = w.kinds[i];
    if (kd == ZB_DF_GZIP) kind = 0;
    else if (kd == ZB_DF_ZLIB) kind = 1;
    else return;
  }
  const uint64_t buflen = w.lens ? w.lens[i] : w.off[i + 1] - w.off[i];
  const uint32_t p0 = w.first[i];
  const uint32_t np = (uint32_t)((buflen + CK_PIECE - 1) / CK_PIECE);
  if (np <= w.big_pieces) return;  // k_buffer_combine's
  const uint32_t t = threadIdx.x;
  uint32_t r = 0;
  uint64_t a = 0, b = 0, end = 0;
  if (kind == 0) {
    uint32_t step = 0;
    for (uint32_t k = t; k < np; k += CKB_THREADS) {
      const uint32_t l = piece_len(buflen, (uint64_t)k * CK_PIECE);
      const uint32_t raw = w.piece_out[p0 + k].crc_raw;
      if (k >= CKB_THREADS) {
        if (l == CK_PIECE) {
          if (!step) step = zb_xpow8_t(w.tabs->pow2, (uint64_t)CKB_THREADS * CK_PIECE);
          r = zb_gf2_mul(r, step);
        } else {
          r = zb_gf2_mul(r, zb_xpow8_t(w.tabs->pow2, (uint64_t)(CKB_THREADS - 1) * CK_PIECE + l));
        }
      }
      r ^= raw;
      end = (uint64_t)k * CK_PIECE + l;
    }
    if (t < np && end < buflen) r = zb_gf2_mul(r, zb_xpow8_t(w.tabs->pow2, buflen - end));
    r = zb_warp_xor(r);
  } else {
    for (uint32_t k = t; k < np; k += CKB_THREADS) {
      const uint32_t l = piece_len(buflen, (uint64_t)k * CK_PIECE);
      const uint32_t ab = w.piece_out[p0 + k].adler;
      const uint64_t ak = ab & 0xffffu, bk = ab >> 16;
      const uint64_t after = (buflen - ((uint64_t)k * CK_PIECE + l)) % ZB_ADLER_MOD;
      a += ak;
      b = (b + bk + after * ak) % ZB_ADLER_MOD;
    }
    a = zb_warp_sum64(a % ZB_ADLER_MOD);
    b = zb_warp_sum64(b);
  }
  if ((t & 31u) == 0) {
    red_r[t >> 5] = r;
    red_a[t >> 5] = a;
    red_b[t >> 5] = b;
  }
  __syncthreads();
  if (t != 0) return;
  r = 0;
  a = b = 0;
  for (int j = 0; j < CKB_THREADS / 32; j++) {
    r ^= red_r[j];
    a += red_a[j];
    b += red_b[j];
  }
  ck_finish(w, i, kind, r, a, b, buflen);
}

// ------------------------------------------------------------------------------------
// Candidate segment boundaries of a large member (see zb_kernels.h).
__global__ void __launch_bounds__(256) k_find_sync(const uint8_t *src, uint64_t lo, uint64_t hi, uint64_t *out, uint32_t cap,
                                                   uint32_t *count) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t p = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p + 4 <= hi; p += stride) {
    if (src[p + 2] == 0xffu && src[p + 3] == 0xffu && src[p] == 0u && src[p + 1] == 0u) {
      const uint32_t k = atomicAdd(count, 1u);
      if (k < cap) out[k] = p + 4;
    }
  }
}

// ------------------------------------------------------------------------------------
// Speculative segments of ONE large raw-deflate stream (SURVEY 8f-1; the reference decodes any stream
// at 0.5-1.6 GB/s on a CPU core, inflate.nim:173-250 -- a single 8-lane group here is ~50x slower, so a
// large foreign member has to be cut).  A stream can only be entered at a block boundary, and nothing
// in it says where those are: k_find_blocks tests EVERY bit offset of the payload for a plausible
// dynamic-block header (BTYPE = 2, HLIT/HDIST in range, a COMPLETE code-length code, code lengths that
// parse to exactly HLIT + HDIST entries, a complete literal/length code that can encode end-of-block,
// a distance code that is not over-subscribed).  Random data passes with vanishing probability, and a
// false candidate is caught later anyway: the decode of the previous segment must END exactly on it.
__device__ __forceinline__ uint64_t fb_ld64(const uint8_t *src, uint64_t byte, uint64_t limit) {
  uint64_t v = 0;
#pragma unroll
  for (int k = 0; k < 8; k++)
    if (byte + (uint64_t)k < limit) v |= (uint64_t)src[byte + (uint64_t)k] << (8 * k);
  return v;
}
// up to 32 bits at absolute bit position `bit`
__device__ __forceinline__ uint32_t fb_bits(const uint8_t *src, uint64_t bit, uint64_t limit_byte) {
  const uint64_t w = fb_ld64(src, bit >> 3, limit_byte);
  return (uint32_t)(w >> (bit & 7ull));
}

__device__ bool fb_full_check(const uint8_t *src, uint64_t bit, uint64_t limit_byte) {
  const uint8_t order[19] = ZB_CLCL_ORDER;
  uint32_t hdr = fb_bits(src, bit, limit_byte);
  const int hlit = (int)((hdr >> 3) & 31u) + 257, hdist = (int)((hdr >> 8) & 31u) + 1, hclen = (int)((hdr >> 13) & 15u) + 4;
  uint64_t pos = bit + 17;
  uint8_t cl[19];
  for (int i = 0; i < 19; i++) cl[i] = 0;
  for (int i = 0; i < hclen; i++, pos += 3) cl[order[i]] = (uint8_t)(fb_bits(src, pos, limit_byte) & 7u);
  // canonical code-length code -> 128-entry lookup: symbol | len << 5
  uint8_t tab[128];
  for (int i = 0; i < 128; i++) tab[i] = 0;
  {
    uint32_t count[8] = {0, 0, 0, 0, 0, 0, 0, 0}, next[8];
    for (int i = 0; i < 19; i++) count[cl[i]]++;
    count[0] = 0;
    uint32_t code = 0;
    for (int l = 1; l < 8; l++) {
      code = (code + count[l - 1]) << 1;
      next[l] = code;
    }
    for (int sy = 0; sy < 19; sy++) {
      const int l = cl[sy];
      if (!l) continue;
      const uint32_t c = next[l]++;
      const uint32_t rev = __brev(c) >> (32 - l);
      for (uint32_t idx = rev; idx < 128u; idx += 1u << l) tab[idx] = (uint8_t)(sy | (l << 5));
    }
  }
  uint8_t lens[320];
  const int total = hlit + hdist;
  int i = 0;
  uint32_t prev = 0;
  while (i < total) {
    if ((pos >> 3) >= limit_byte) return false;
    const uint32_t x = fb_bits(src, pos, limit_byte);
    const uint32_t e = tab[x & 127u];
    const uint32_t l = e >> 5, sym = e & 31u;
    if (l == 0) return false;
    pos += l;
    const uint32_t y = x >> l;
    if (sym <= 15) {
      lens[i++] = (uint8_t)sym;
      prev = sym;
    } else {
      int rep;
      uint32_t v = 0;
      if (sym == 16) {
        if (i == 0) return false;
        rep = 3 + (int)(y & 3u);
        pos += 2;
        v = prev;
      } else if (sym == 17) {
        rep = 3 + (int)(y & 7u);
        pos += 3;
        prev = 0;
      } else {
        rep = 11 + (int)(y & 127u);
        pos += 7;
        prev = 0;
      }
      if (i + rep > total) return false;
      for (int k = 0; k < rep; k++) lens[i++] = (uint8_t)v;
    }
  }
  if (lens[256] == 0) return false;  // end-of-block must have a code
  uint32_t kl = 0, kd = 0, nd = 0;
  for (int k = 0; k < hlit; k++)
    if (lens[k]) kl += 32768u >> lens[k];
  for (int k = 0; k < hdist; k++)
    if (lens[hlit + k]) {
      kd += 32768u >> lens[hlit + k];
      nd++;
    }
  if (kl != 32768u) return false;                 // every encoder emits a complete literal/length code
  if (kd > 32768u) return false;                  // over-subscribed
  if (kd != 32768u && nd > 1) return false;       // incomplete only in the one-code (or no-code) case
  return true;
}

__global__ void __launch_bounds__(256) k_find_blocks(const uint8_t *src, uint64_t lo_bit, uint64_t hi_bit, uint64_t limit_byte,
                                                     uint64_t *out, uint32_t cap, uint32_t *count) {
  const uint8_t order[19] = ZB_CLCL_ORDER;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t bit = lo_bit + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; bit + 80 <= hi_bit; bit += stride) {
    // the 17 fixed header bits + 19 x 3 bits of code-length code lengths live in 74 bits
    const uint64_t byte = bit >> 3;
    const uint32_t sh = (uint32_t)(bit & 7ull);
    const uint64_t w0 = fb_ld64(src, byte, limit_byte), w1 = fb_ld64(src, byte + 8, limit_byte);
    const uint64_t a = sh ? (w0 >> sh) | (w1 << (64 - sh)) : w0;   // bits 0..63 from `bit`
    const uint32_t b = (uint32_t)(w1 >> sh);                        // bits 64..
    if (((a >> 1) & 3ull) != 2ull) continue;          // BTYPE = dynamic
    if (((a >> 3) & 31ull) > 29ull) continue;         // HLIT <= 286 - 257
    if (((a >> 8) & 31ull) > 29ull) continue;         // HDIST <= 30 - 1
    const int hclen = (int)((a >> 13) & 15ull) + 4;
    uint32_t kraft = 0;
    bool len_ok = true;
#pragma unroll
    for (int i = 0; i < 19; i++) {
      const int p = 17 + 3 * i;
      const uint32_t l = p + 3 <= 64 ? (uint32_t)(a >> p) & 7u : p >= 64 ? (b >> (p - 64)) & 7u
                                     : (uint32_t)((a >> p) | ((uint64_t)b << (64 - p))) & 7u;
      if (i < hclen && l) kraft += 128u >> l;
      (void)order;
    }
    if (!len_ok || kraft != 128u) continue;           // the code-length code must be complete
    if (!fb_full_check(src, bit, limit_byte)) continue;
    const uint32_t k = atomicAdd(count, 1u);
    if (k < cap) out[k] = bit;
  }
}

cudaError_t zb_launch_find_blocks(const uint8_t *src, uint64_t lo_bit, uint64_t hi_bit, uint64_t limit_byte, uint64_t *out,
                                  uint32_t cap, uint32_t *count, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  if (hi_bit < lo_bit + 80) return cudaSuccess;
  uint64_t blocks = (hi_bit - lo_bit + 255) / 256;
  const uint64_t max_blocks = 64ull * (uint64_t)zb_sm_count();
  if (blocks > max_blocks) blocks = max_blocks;
  k_find_blocks<<<(uint32_t)blocks, 256, 0, s>>>(src, lo_bit, hi_bit, limit_byte, out, cap, count);
  return cudaGetLastError();
}

// ---- markers -> bytes ----
// Segment i was decoded into scr[soff[i] ...) as uint16 symbols: < 256 a byte, 0x8000 | k byte k of the
// 32768 bytes that precede the segment in the member's output.  (1) k_mark_prefill puts those marker
// symbols in front of every segment before the decode, so that a copy reaching before the segment's start
// simply copies markers.  (2) k_resolve_tails walks the segments IN ORDER with the last 32 KiB of resolved
// output in a shared-memory ring and finalises the last min(n, 32768) bytes of every segment -- exactly
// the bytes the following segments' markers can refer to.  (3) k_resolve_rest then resolves everything
// else in parallel, reading windows from the finished tails in dst.
struct ZbMarkSeg {
  uint64_t scr;   // element offset of the segment's first output symbol in the scratch
  uint64_t dst;   // byte offset of the segment's first output byte in dst
  uint32_t n;     // output bytes
  uint32_t pad;
};
__global__ void __launch_bounds__(256) k_mark_prefill(uint16_t *scr, const ZbMarkSeg *segs) {
  const ZbMarkSeg sg = segs[blockIdx.y];
  const uint32_t k = blockIdx.x * 256u + threadIdx.x;
  if (k < 32768u) scr[sg.scr - 32768ull + k] = (uint16_t)(0x8000u | k);
}

#define RT_THREADS 1024
#define RT_PER (32768 / RT_THREADS)
__global__ void __launch_bounds__(RT_THREADS, 1) k_resolve_tails(const uint16_t *scr, const ZbMarkSeg *segs, uint32_t nseg,
                                                                 uint8_t *dst, int *bad) {
  extern __shared__ uint8_t ring[];   // ring[p & 32767] = resolved output byte at member position p (relative to segs[0].dst)
  const uint32_t tid = threadIdx.x;
  const uint64_t base = segs[0].dst;
  for (uint32_t i = 0; i < nseg; i++) {
    const ZbMarkSeg sg = segs[i];
    const uint32_t T = min(sg.n, 32768u), j0 = sg.n - T;
    const uint64_t p0 = sg.dst - base;          // member position of the segment's first byte
    uint8_t val[RT_PER];
    bool any_bad = false;
#pragma unroll
    for (int r = 0; r < RT_PER; r++) {
      const uint32_t j = j0 + tid + (uint32_t)r * RT_THREADS;
      val[r] = 0;
      if (j < sg.n) {
        const uint32_t sy = scr[sg.scr + j];
        if (sy < 256u) val[r] = (uint8_t)sy;
        else {
          // marker k = byte at member position p0 - 32768 + k; it must exist (a reference before the
          // start of the whole stream is the reference's "distance > op" error, inflate.nim:224)
          const uint32_t k = sy & 0x7fffu;
          if (p0 + k < 32768ull) any_bad = true;
          val[r] = ring[(uint32_t)(p0 + k) & 32767u];
        }
      }
    }
    __syncthreads();   // every read of the old window is done before it is overwritten
#pragma unroll
    for (int r = 0; r < RT_PER; r++) {
      const uint32_t j = j0 + tid + (uint32_t)r * RT_THREADS;
      if (j < sg.n) {
        ring[(uint32_t)(p0 + j) & 32767u] = val[r];
        dst[sg.dst + j] = val[r];
      }
    }
    if (any_bad) *bad = 1;
    __syncthreads();
  }
}

// base: dst offset of the member's first output byte (markers before it are the "distance too far back" error)
__global__ void __launch_bounds__(256) k_resolve_rest(const uint16_t *scr, const ZbMarkSeg *segs, uint32_t nseg, uint32_t slabs,
                                                      uint64_t base, uint8_t *dst, int *bad) {
  for (uint64_t b = blockIdx.x; b < (uint64_t)nseg * slabs; b += gridDim.x) {
    const ZbMarkSeg sg = segs[b / slabs];
    const uint32_t x = (uint32_t)(b % slabs);
    const uint64_t p0 = sg.dst - base;   // member position of the segment's first byte
    const uint32_t T = min(sg.n, 32768u), rest = sg.n - T;
    for (uint32_t j = x * 2048u + threadIdx.x; j < min(rest, x * 2048u + 2048u); j += 256u) {
      const uint32_t sy = scr[sg.scr + j];
      uint8_t v = (uint8_t)sy;
      if (sy >= 256u) {
        const uint32_t k = sy & 0x7fffu;
        if (p0 + k < 32768ull) {   // before the start of the stream: the member goes to the serial decode
          *bad = 1;
          v = 0;
        } else {
          v = dst[sg.dst - 32768ull + k];
        }
      }
      dst[sg.dst + j] = v;
    }
  }
}

// ---- the parallel window resolve (segments at this library's sync joints, zb_api.cu: inflate_member_joints) ----
// The per-element rules and the three steps are described in zb_resolve.h.  The segments of one launch are a
// window of a member; its groups are gsz consecutive segments each.
// (A) one CTA per group: tails in place as "byte or marker into the group's incoming window", the group's
//     outgoing window map to gmap[group].
__global__ void __launch_bounds__(RT_THREADS, 1) k_resolve_groups(uint16_t *scr, const ZbMarkSeg *segs, uint32_t nseg,
                                                                  uint32_t gsz, uint64_t base, uint16_t *gmap, int *bad) {
  extern __shared__ uint16_t rring[];   // rring[zb_rs_slot(p)] = symbol at member position p
  const uint32_t tid = threadIdx.x, s0 = blockIdx.x * gsz, s1 = min(nseg, s0 + gsz);
  const uint64_t q0 = segs[s0].dst - base;
  for (uint32_t k = tid; k < ZB_RS_WIN; k += RT_THREADS) rring[zb_rs_slot(q0 + k)] = zb_rs_incoming(k);
  __syncthreads();
  bool any_bad = false;
  for (uint32_t i = s0; i < s1; i++) {
    const ZbMarkSeg sg = segs[i];
    const uint32_t T = min(sg.n, ZB_RS_WIN), j0 = sg.n - T;
    const uint64_t p0 = sg.dst - base;
    uint16_t *tail = scr + sg.scr + j0;
    uint32_t val[RT_PER / 2];   // two symbols per register (no spills at 1024 threads)
#pragma unroll
    for (int r = 0; r < RT_PER; r++) {
      const uint32_t k = tid + (uint32_t)r * RT_THREADS;
      const uint32_t v = k < T ? zb_rs_ring_lookup(tail[k], p0, rring, any_bad) : 0u;
      val[r / 2] = (r & 1) ? (val[r / 2] | (v << 16)) : v;
    }
    __syncthreads();   // every read of the old window is done before it is overwritten
#pragma unroll
    for (int r = 0; r < RT_PER; r++) {
      const uint32_t k = tid + (uint32_t)r * RT_THREADS;
      if (k < T) {
        const uint16_t v = (uint16_t)((r & 1) ? (val[r / 2] >> 16) : val[r / 2]);
        rring[zb_rs_slot(p0 + j0 + k)] = v;
        tail[k] = v;
      }
    }
    __syncthreads();
  }
  const uint64_t q1 = segs[s1 - 1].dst + segs[s1 - 1].n - base;   // one past the group's last position
  for (uint32_t k = tid; k < ZB_RS_WIN; k += RT_THREADS) gmap[(uint64_t)blockIdx.x * ZB_RS_WIN + k] = rring[zb_rs_slot(q1 + k)];
  if (any_bad) *bad = 1;
}

// (B) one CTA: the incoming window of every group, in order.  The window's own incoming window is the resolved
// output in front of member position w0 (positions before the member start read as 0: markers there set bad in (A)).
__global__ void __launch_bounds__(RT_THREADS, 1) k_resolve_compose(const uint16_t *gmap, uint32_t ngroups, const uint8_t *dst,
                                                                   uint64_t base, uint64_t w0, uint8_t *gin) {
  __shared__ uint8_t win[ZB_RS_WIN];
  const uint32_t tid = threadIdx.x;
  for (uint32_t k = tid; k < ZB_RS_WIN; k += RT_THREADS) win[k] = w0 + k >= ZB_RS_WIN ? dst[base + w0 + k - ZB_RS_WIN] : (uint8_t)0;
  __syncthreads();
  for (uint32_t g = 0; g < ngroups; g++) {
    const uint16_t *m = gmap + (uint64_t)g * ZB_RS_WIN;
    uint8_t *in = gin + (uint64_t)g * ZB_RS_WIN;
    uint8_t v[RT_PER];
#pragma unroll
    for (int r = 0; r < RT_PER; r++) {
      const uint32_t k = tid + (uint32_t)r * RT_THREADS;
      in[k] = win[k];
      v[r] = zb_rs_compose(m[k], win);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RT_PER; r++) win[tid + (uint32_t)r * RT_THREADS] = v[r];
    __syncthreads();
  }
}

// (C) every tail symbol against its group's incoming window -> dst
__global__ void __launch_bounds__(256) k_resolve_tails_par(const uint16_t *scr, const ZbMarkSeg *segs, uint32_t nseg,
                                                           uint32_t gsz, const uint8_t *gin, uint8_t *dst) {
  const uint64_t total = (uint64_t)nseg * ZB_RS_WIN, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const uint32_t i = (uint32_t)(t / ZB_RS_WIN), jt = (uint32_t)(t % ZB_RS_WIN);
    const ZbMarkSeg sg = segs[i];
    const uint32_t T = min(sg.n, ZB_RS_WIN);
    if (jt >= T) continue;
    const uint32_t j = sg.n - T + jt;
    dst[sg.dst + j] = zb_rs_compose(scr[sg.scr + j], gin + (uint64_t)(i / gsz) * ZB_RS_WIN);
  }
}

static uint32_t resolve_rest_grid(uint32_t nseg, uint32_t slabs) {
  return (uint32_t)std::min<uint64_t>((uint64_t)nseg * slabs, 64ull * (uint64_t)zb_sm_count());
}

cudaError_t zb_launch_mark_prefill(uint16_t *scr, const void *segs, uint32_t nseg, cudaStream_t s) {
  if (!nseg) return cudaSuccess;
  k_mark_prefill<<<dim3(128, nseg), 256, 0, s>>>(scr, (const ZbMarkSeg *)segs);
  return cudaGetLastError();
}
cudaError_t zb_launch_resolve(const uint16_t *scr, const void *segs, uint32_t nseg, uint32_t max_n, uint64_t base, uint8_t *dst,
                              int *bad, cudaStream_t s) {
  if (!nseg) return cudaSuccess;
  k_resolve_tails<<<1, RT_THREADS, 32768, s>>>(scr, (const ZbMarkSeg *)segs, nseg, dst, bad);
  const uint32_t slabs = (max_n + 2047u) / 2048u;
  if (slabs) k_resolve_rest<<<resolve_rest_grid(nseg, slabs), 256, 0, s>>>(scr, (const ZbMarkSeg *)segs, nseg, slabs, base, dst, bad);
  return cudaGetLastError();
}

cudaError_t zb_launch_resolve_groups(uint16_t *scr, const void *segs, uint32_t nseg, uint32_t max_n, uint32_t gsz, uint64_t base,
                                     uint64_t w0, uint16_t *gmap, uint8_t *gin, uint8_t *dst, int *bad, cudaStream_t s) {
  if (!nseg) return cudaSuccess;
  const ZbMarkSeg *sg = (const ZbMarkSeg *)segs;
  const uint32_t ngroups = (nseg + gsz - 1) / gsz;
  k_resolve_groups<<<ngroups, RT_THREADS, ZB_RS_WIN * 2, s>>>(scr, sg, nseg, gsz, base, gmap, bad);
  k_resolve_compose<<<1, RT_THREADS, 0, s>>>(gmap, ngroups, dst, base, w0, gin);
  const uint32_t tgrid = (uint32_t)std::min<uint64_t>(((uint64_t)nseg * ZB_RS_WIN + 255) / 256, 64ull * (uint64_t)zb_sm_count());
  k_resolve_tails_par<<<tgrid, 256, 0, s>>>(scr, sg, nseg, gsz, gin, dst);
  const uint32_t slabs = (max_n + 2047u) / 2048u;
  if (slabs) k_resolve_rest<<<resolve_rest_grid(nseg, slabs), 256, 0, s>>>(scr, sg, nseg, slabs, base, dst, bad);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) k_gather(const uint8_t *src, const ZbGather *gs, void *dst) {
  const ZbGather g = gs[blockIdx.x];
  const uint8_t *s = src + g.src;
  if (g.wide) {
    uint16_t *d = reinterpret_cast<uint16_t *>(dst) + g.dst;
    for (uint32_t k = threadIdx.x; k < g.n; k += 256u) d[k] = s[k];
  } else {
    uint8_t *d = reinterpret_cast<uint8_t *>(dst) + g.dst;
    for (uint32_t k = threadIdx.x; k < g.n; k += 256u) d[k] = s[k];
  }
}
cudaError_t zb_launch_gather(const uint8_t *src, const ZbGather *g, uint32_t n, void *dst, cudaStream_t s) {
  if (!n) return cudaSuccess;
  k_gather<<<n, 256, 0, s>>>(src, g, dst);
  return cudaGetLastError();
}

cudaError_t zb_launch_find_sync(const uint8_t *src, uint64_t lo, uint64_t hi, uint64_t *out, uint32_t cap,
                                uint32_t *count, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(count, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  if (hi < lo + 4) return cudaSuccess;
  uint64_t blocks = (hi - lo + 255) / 256;
  const uint64_t max_blocks = 16ull * (uint64_t)zb_sm_count();
  if (blocks > max_blocks) blocks = max_blocks;
  k_find_sync<<<(uint32_t)blocks, 256, 0, s>>>(src, lo, hi, out, cap, count);
  return cudaGetLastError();
}

// function attributes are per device: zb200_init calls this once for the ctx's device
cudaError_t zb_setup_inflate_attrs() {
  const int smem = (int)(INF_GROUPS * sizeof(GroupSmem)) + 256;
  cudaError_t e = cudaFuncSetAttribute(k_inflate<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_inflate<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_inflate<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_inflate<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_inflate<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_resolve_tails, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_resolve_groups, cudaFuncAttributeMaxDynamicSharedMemorySize, ZB_RS_WIN * 2);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_piece_checksum<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CK_SM_TOTAL);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_piece_checksum<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CK_SM_TOTAL_ADLER);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_piece_checksum<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  // Load every kernel NOW (CUDA loads a function lazily at its first launch, and that load can wait for the device
  // to go idle): a launch queued behind the gated inflate kernel must not be the one that triggers it -- the kernel
  // would be waiting for copies this thread has not queued yet.
  cudaFuncAttributes fa;
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_buffer_combine);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_piece_fold);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_buffer_combine_big);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_find_sync);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_find_blocks);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_mark_prefill);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_resolve_rest);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_resolve_compose);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_resolve_tails_par);
  return e;
}

cudaError_t zb_launch_inflate(const ZbInflateWork &w, cudaStream_t s) {
  if (w.n == 0) return cudaSuccess;
  const int smem = (int)(INF_GROUPS * sizeof(GroupSmem)) + 256;
  const int sms = zb_sm_count();
  uint32_t per_sm = (uint32_t)((227 * 1024) / (smem + 1024));
  if (per_sm < 1) per_sm = 1;
  uint32_t blocks = (uint32_t)sms * per_sm;
  uint32_t need = (w.n + INF_GROUPS - 1) / INF_GROUPS;
  if (blocks > need) blocks = need;
  cudaError_t e = cudaMemsetAsync(w.counter, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  if (w.mdict && !w.seg_bits) {
    if (w.count_only) k_inflate<true, false, true><<<blocks, INF_THREADS, smem, s>>>(w);
    else k_inflate<false, false, true><<<blocks, INF_THREADS, smem, s>>>(w);
  } else if (w.count_only) k_inflate<true, false><<<blocks, INF_THREADS, smem, s>>>(w);
  else if (w.mark) k_inflate<false, true><<<blocks, INF_THREADS, smem, s>>>(w);
  else k_inflate<false, false><<<blocks, INF_THREADS, smem, s>>>(w);
  return cudaGetLastError();
}

cudaError_t zb_launch_checksum(const ZbChecksumWork &w, cudaStream_t s) {
  if (w.n == 0) return cudaSuccess;
  const int sms = zb_sm_count();
  if (w.n_pieces) {
    if (!w.kinds && w.kind == 1) {  // Adler-32 throughout: the table-free instantiation, three CTAs per SM
      const uint32_t grid = std::min<uint32_t>(3u * (uint32_t)sms, w.n_pieces);
      k_piece_checksum<true><<<grid, CK_THREADS_ADLER, CK_SM_TOTAL_ADLER, s>>>(w);
    } else {
      const uint32_t grid = std::min<uint32_t>((uint32_t)sms, w.n_pieces);
      k_piece_checksum<false><<<grid, CK_THREADS, CK_SM_TOTAL, s>>>(w);
      k_piece_fold<<<std::min<uint32_t>((w.n_pieces + 7) / 8, 8u * (uint32_t)sms), 256, 0, s>>>(w);
    }
  }
  k_buffer_combine<<<(w.n + 3) / 4, 128, 0, s>>>(w);
  if (w.big_pieces) k_buffer_combine_big<<<w.n, CKB_THREADS, 0, s>>>(w);
  return cudaGetLastError();
}
