// zb_resolve.h -- per-element rules of the parallel window resolve (host + device).
//
// Segments of one member decoded as uint16 symbols (ZbInflateWork::mark): a symbol < 256 is a byte, 0x8000 | k
// stands for byte k of the 32768 bytes in front of the segment.  The resolve in zb_inflate.cu works in three
// steps over groups of consecutive segments:
//   (A) one CTA per group walks its segments in order with a ring of the last 32768 symbols.  The ring starts
//       as the group's INCOMING window: position q0 - 32768 + k holds the marker 0x8000 | k (q0: the group's
//       first output position).  A marker of a segment is looked up in the ring (zb_rs_ring_lookup), so every
//       tail symbol ends up as a byte or a marker into the group's incoming window; at the end the ring is the
//       group's outgoing window map, in the same terms.
//   (B) one CTA composes the groups in order: incoming window of group g + 1 = map of group g applied to the
//       incoming window of group g (zb_rs_compose) -- G x 32768 lookups instead of S x 32768.
//   (C) every tail symbol is composed with its group's incoming window, in parallel.
// The same functions run on the CPU in tests/native/resolve_units.cpp against a plain sequential resolve.
#pragma once
#include "zb_common.h"

#define ZB_RS_WIN 32768u

// ring slot of member output position p (positions before the member start are never read: see below)
ZB_HD uint32_t zb_rs_slot(uint64_t p) { return (uint32_t)(p & (ZB_RS_WIN - 1u)); }

// The incoming-window marker that a group whose first output position is q0 keeps in the ring slot of position
// q0 - 32768 + k.
ZB_HD uint16_t zb_rs_incoming(uint32_t k) { return (uint16_t)(0x8000u | k); }

// Symbol sy of a segment whose first output position is p0 (member-relative), resolved through a ring that holds
// the symbols of the 32768 positions before the symbol's segment.  A marker that points before the start of the
// member is the reference's "distance too far back" error: bad is set (the member goes to the serial decode).
ZB_HD uint16_t zb_rs_ring_lookup(uint16_t sy, uint64_t p0, const uint16_t *ring, bool &bad) {
  if (sy < 256u) return sy;
  const uint32_t k = sy & 0x7fffu;
  if (p0 + k < (uint64_t)ZB_RS_WIN) bad = true;
  return ring[zb_rs_slot(p0 + k)];   // position p0 - 32768 + k
}

// A symbol in terms of a group's incoming window -> the byte, given that window's bytes.
ZB_HD uint8_t zb_rs_compose(uint16_t sy, const uint8_t *win) { return sy < 256u ? (uint8_t)sy : win[sy & 0x7fffu]; }
