// TEST INFRASTRUCTURE ONLY -- never part of libzopfli.so.
//
// The host mock of tests/hostmock (an oracle-backed stand-in for zb::Engine) with parse ranges that honour
// ParseRange::floor, as the engine does: a range with a floor is the oracle's parse of in + floor, positions
// shifted by the floor (squeeze.c:229-230 on the shifted input: the window starts at max(instart - 32768,
// floor)).  The symbols do not depend on where their range starts, so they land at their absolute positions
// unchanged.  tests/floormock/Makefile links it with the product's host sources into
// tests/_build/libzopfli_floormock.so for the restart-point tests, whose waves hold units above different
// floors.  The mock's source is compiled here as it stands: its oracle calls are routed through the wrappers
// below, which find the floor in the ParseRange whose instart the call passes (every call passes r[i].instart).
#include <stddef.h>

#include "../../oracle/zopfli_oracle.h"
#include "../../zopfli_b200/csrc/engine.hpp"

namespace {

const zb::ParseRange& range_of(const uint64_t& instart) {  // instart is the member of a ParseRange
  return *reinterpret_cast<const zb::ParseRange*>(reinterpret_cast<const char*>(&instart) -
                                                   offsetof(zb::ParseRange, instart));
}

void floor_greedy(const uint8_t* in, const uint64_t& instart, uint64_t inend, ZoStore* out) {
  const uint64_t f = range_of(instart).floor;
  zo_lz77_greedy(in + f, instart - f, inend - f, out);
}

void floor_optimal(const uint8_t* in, const uint64_t& instart, uint64_t inend, int numiterations, ZoStore* out) {
  const uint64_t f = range_of(instart).floor;
  zo_lz77_optimal(in + f, instart - f, inend - f, numiterations, out);
}

void floor_optimal_fixed(const uint8_t* in, const uint64_t& instart, uint64_t inend, ZoStore* out) {
  const uint64_t f = range_of(instart).floor;
  zo_lz77_optimal_fixed(in + f, instart - f, inend - f, out);
}

// a start that is not a ParseRange's member (a temporary) has no range to take the floor from: refused at compile
// time rather than read from the wrong memory
void floor_greedy(const uint8_t*, const uint64_t&&, uint64_t, ZoStore*) = delete;
void floor_optimal(const uint8_t*, const uint64_t&&, uint64_t, int, ZoStore*) = delete;
void floor_optimal_fixed(const uint8_t*, const uint64_t&&, uint64_t, ZoStore*) = delete;

}  // namespace

#define zo_lz77_greedy floor_greedy
#define zo_lz77_optimal floor_optimal
#define zo_lz77_optimal_fixed floor_optimal_fixed
#include "../hostmock/mock_engine.cpp"
