// tests/sim/search_probe.cc -- TEST INFRASTRUCTURE (tests/test_search_probe.py).  The product's br_debug_search hook on the
// sim's index: one match search per probe (brotli_b200/csrc/br_probe.h) with a one-lane warp, from the state the caller
// specifies.  Same arguments as br_debug_search (br_kernels.cu); it runs the search once, with the pipeline's row grouping.
#include "br_sim.cc"
#include "../../brotli_b200/csrc/br_probe.h"

extern "C" int sim_debug_search(int quality, int lgwin, int lgblock, u32 size_hint, const u8* in, u32 n, const u32* bounds,
                                u32 nstreams, const u32* snap, const u32* own_in, u32 heavy_min, const u32* probes, u32 np,
                                u32* res) {
  if (n == 0 || nstreams == 0 || bounds[nstreams - 1] != n) return 0;
  std::vector<u32> kinds(nstreams, 3);
  const BrCuts c = {bounds, kinds.data(), nstreams - 1, 1, 1, 0, nullptr, lgblock, 0, 0, nullptr};
  SimStream* m = sim_setup(quality, lgwin, size_hint, in, n, &c);
  if (!m) return 0;
  BrStream& s = m->s;
  if (heavy_min) s.P.heavy_min = heavy_min;
  const u32 nw = (n + 31) / 32;
  std::fill(m->bits_latest.begin(), m->bits_latest.end(), 0);
  std::copy(snap, snap + nw, m->bits_latest.begin());
  std::vector<u32> own(m->bits_latest.size(), 0);
  std::copy(own_in, own_in + nw, own.begin());
  sim_build_storedS(*m);
  for (u32 t = 0; t < np; ++t) {
    const u32* pr = probes + (size_t)t * BR_PROBE_WORDS;
    u32* r = res + (size_t)t * BR_PROBE_WORDS;
    br_walk_dispatch(s.P, [&](auto g, auto) { br_probe_search<decltype(g)::value>(s, own.data(), pr, r); });
  }
  delete m;
  return 1;
}
