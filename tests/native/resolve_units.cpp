// CPU model of the parallel window resolve (zippy_b200/csrc/zb_resolve.h), built as a shared library for
// tests/test_resolve_units.py: the three steps of zb_inflate.cu (k_resolve_groups, k_resolve_compose,
// k_resolve_tails_par + k_resolve_rest) written with the header's per-element rules, and a plain sequential
// resolve to compare them with.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../zippy_b200/csrc/zb_resolve.h"

// Input of both: the symbols of nseg consecutive segments of one window (segment i has n[i] symbols, stored one
// after another in sym), the window's first member position w0, and prev = the 32768 output bytes in front of w0
// (only the ones at member positions >= 0 are read).  out gets the window's bytes; the return value is the bad flag.
extern "C" int t_resolve_seq(const uint16_t *sym, const uint32_t *n, uint32_t nseg, uint64_t w0, const uint8_t *prev,
                             uint8_t *out) {
  int bad = 0;
  uint64_t o = 0;
  for (uint32_t i = 0; i < nseg; i++) {
    const uint64_t p0 = w0 + o;   // member position of the segment's first byte
    for (uint32_t j = 0; j < n[i]; j++) {
      const uint16_t sy = sym[o + j];
      if (sy < 256) {
        out[o + j] = (uint8_t)sy;
        continue;
      }
      const uint64_t k = sy & 0x7fffu;
      if (p0 + k < 32768) {   // before the member start
        bad = 1;
        out[o + j] = 0;
        continue;
      }
      const uint64_t p = p0 + k - 32768;   // the member position the marker stands for
      out[o + j] = p >= w0 ? out[p - w0] : prev[p - (w0 - 32768)];
    }
    o += n[i];
  }
  return bad;
}

extern "C" int t_resolve_groups(const uint16_t *sym_in, const uint32_t *n, uint32_t nseg, uint32_t gsz, uint64_t w0,
                                const uint8_t *prev, uint8_t *out) {
  std::vector<uint64_t> off(nseg + 1, 0);
  for (uint32_t i = 0; i < nseg; i++) off[i + 1] = off[i] + n[i];
  std::vector<uint16_t> sym(sym_in, sym_in + off[nseg]);
  const uint32_t ng = (nseg + gsz - 1) / gsz;
  std::vector<uint16_t> gmap((size_t)ng * ZB_RS_WIN);
  bool bad = false;
  // (A) per group: the tails in place, the outgoing window map
  for (uint32_t g = 0; g < ng; g++) {
    const uint32_t s0 = g * gsz, s1 = s0 + gsz < nseg ? s0 + gsz : nseg;
    std::vector<uint16_t> ring(ZB_RS_WIN);
    const uint64_t q0 = w0 + off[s0];
    for (uint32_t k = 0; k < ZB_RS_WIN; k++) ring[zb_rs_slot(q0 + k)] = zb_rs_incoming(k);
    for (uint32_t i = s0; i < s1; i++) {
      const uint32_t T = n[i] < ZB_RS_WIN ? n[i] : ZB_RS_WIN, j0 = n[i] - T;
      const uint64_t p0 = w0 + off[i];
      std::vector<uint16_t> val(T);
      for (uint32_t k = 0; k < T; k++) val[k] = zb_rs_ring_lookup(sym[off[i] + j0 + k], p0, ring.data(), bad);
      for (uint32_t k = 0; k < T; k++) {
        ring[zb_rs_slot(p0 + j0 + k)] = val[k];
        sym[off[i] + j0 + k] = val[k];
      }
    }
    const uint64_t q1 = w0 + off[s1];
    for (uint32_t k = 0; k < ZB_RS_WIN; k++) gmap[(size_t)g * ZB_RS_WIN + k] = ring[zb_rs_slot(q1 + k)];
  }
  // (B) the incoming window of every group
  std::vector<uint8_t> gin((size_t)ng * ZB_RS_WIN), win(ZB_RS_WIN);
  for (uint32_t k = 0; k < ZB_RS_WIN; k++) win[k] = w0 + k >= ZB_RS_WIN ? prev[k] : 0;
  for (uint32_t g = 0; g < ng; g++) {
    memcpy(&gin[(size_t)g * ZB_RS_WIN], win.data(), ZB_RS_WIN);
    std::vector<uint8_t> nw(ZB_RS_WIN);
    for (uint32_t k = 0; k < ZB_RS_WIN; k++) nw[k] = zb_rs_compose(gmap[(size_t)g * ZB_RS_WIN + k], win.data());
    win.swap(nw);
  }
  // (C) the tails, then everything else from the finished output (k_resolve_rest)
  for (uint32_t i = 0; i < nseg; i++) {
    const uint32_t T = n[i] < ZB_RS_WIN ? n[i] : ZB_RS_WIN, j0 = n[i] - T;
    for (uint32_t k = 0; k < T; k++)
      out[off[i] + j0 + k] = zb_rs_compose(sym[off[i] + j0 + k], &gin[(size_t)(i / gsz) * ZB_RS_WIN]);
  }
  for (uint32_t i = 0; i < nseg; i++) {
    const uint32_t T = n[i] < ZB_RS_WIN ? n[i] : ZB_RS_WIN;
    const uint64_t p0 = w0 + off[i];
    for (uint32_t j = 0; j < n[i] - T; j++) {
      const uint16_t sy = sym[off[i] + j];
      if (sy < 256) {
        out[off[i] + j] = (uint8_t)sy;
        continue;
      }
      const uint64_t k = sy & 0x7fffu;
      if (p0 + k < 32768) {
        bad = true;
        out[off[i] + j] = 0;
        continue;
      }
      const uint64_t p = p0 + k - 32768;
      out[off[i] + j] = p >= w0 ? out[p - w0] : prev[p - (w0 - 32768)];
    }
  }
  return bad ? 1 : 0;
}
