// The dropout mask of the package (see PhiloxArgs in kernels.h): Philox4x32-10 (Salmon et al., "Parallel random
// numbers: as easy as 1, 2, 3", SC 2011) keyed by the site's seed, counter (n / 4, offset), word n % 4.  The mask of an
// element is a pure function of (seed, offset, n), so a backward kernel regenerates exactly the forward's mask whatever
// order it visits the elements in.  ops.transformer.dropout_keep_reference is the same rule in torch arithmetic.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace edl {

EDL_DEVICE uint4 philox4x32_10(uint32_t k0, uint32_t k1, uint4 c) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// A site's (seed, offset), read through the graph-safe pointers when the draw was captured
struct PhiloxKey {
  uint32_t k0, k1, o0, o1;
  uint32_t threshold;
  float scale;
};

EDL_DEVICE PhiloxKey philox_key(const PhiloxArgs& a) {
  uint64_t seed = a.seed, off = a.offset;
  if (a.seed_ptr != nullptr) {
    seed = (uint64_t)*a.seed_ptr;
    off = (uint64_t)*a.offset_ptr + a.offset_intragraph;
  }
  return PhiloxKey{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)off, (uint32_t)(off >> 32), a.threshold, a.scale};
}

// the four words of counter group g = n / 4
EDL_DEVICE uint4 philox_group(const PhiloxKey& k, uint64_t g) {
  return philox4x32_10(k.k0, k.k1, make_uint4((uint32_t)g, (uint32_t)(g >> 32), k.o0, k.o1));
}

EDL_DEVICE uint32_t philox_word(const uint4& w, int i) { return i == 0 ? w.x : i == 1 ? w.y : i == 2 ? w.z : w.w; }

// keep bits of elements n (bit 0) and n + 1 (bit 1); one Philox evaluation unless the pair straddles a group
EDL_DEVICE uint32_t dropout_keep2(const PhiloxKey& k, uint64_t n) {
  const uint4 w = philox_group(k, n >> 2);
  const int i = (int)(n & 3);
  const uint32_t b0 = philox_word(w, i) >= k.threshold ? 1u : 0u;
  const uint32_t w1 = i == 3 ? philox_group(k, (n >> 2) + 1).x : philox_word(w, i + 1);
  return b0 | (w1 >= k.threshold ? 2u : 0u);
}

EDL_DEVICE bool dropout_keep(const PhiloxKey& k, uint64_t n) {
  return philox_word(philox_group(k, n >> 2), (int)(n & 3)) >= k.threshold;
}

}  // namespace edl
