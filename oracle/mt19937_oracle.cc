// The filter chain's RandomSampler in its MT19937 mode (sm_filter_chain_set_random_sampler), taken from the standard
// library objects the reference's RandomSampler::Filter calls: std::mt19937 and
// std::uniform_real_distribution<double>(0, 1), built anew per Filter call with the seed its random_device returned.
// Nothing here restates the engine or generate_canonical.
#include <cstdint>
#include <random>

namespace {

// a URBG that replays given 32-bit words, to feed crafted words through the library's own distribution
struct Replay {
  using result_type = uint32_t;
  static constexpr result_type min() { return 0; }
  static constexpr result_type max() { return 0xffffffffu; }
  const uint32_t* w;
  result_type operator()() { return *w++; }
};

}  // namespace

extern "C" {

// raw words 0 .. count - 1 of std::mt19937(seed)
int sm_oracle_mt19937_words(uint32_t seed, int64_t count, uint32_t* out) {
  if (count < 0 || (count > 0 && !out)) return -1;
  std::mt19937 eng(seed);
  for (int64_t i = 0; i < count; ++i) out[i] = (uint32_t)eng();
  return 0;
}

// uniform_real_distribution<double>(0, 1) over the words w[0 .. 2n - 1] as an engine would return them -> u[n], and
// keep[j] = u[j] <= rate (the float rate promoted to double, filter_random_sample.cc's test)
int sm_oracle_mt19937_draws(const uint32_t* words_2n, int64_t n, float rate, double* u, uint8_t* keep) {
  if (n < 0 || (n > 0 && (!words_2n || !u || !keep))) return -1;
  Replay eng{words_2n};
  std::uniform_real_distribution<> distr(0., 1.);
  for (int64_t j = 0; j < n; ++j) {
    u[j] = distr(eng);
    keep[j] = u[j] <= rate ? 1 : 0;
  }
  return eng.w == words_2n + 2 * n ? 0 : -2;   // two words per draw
}

// RandomSampler::Filter over n points with std::mt19937 seeded `seed`: keep[j] = 1 for the kept points; a rate above
// 0.999 keeps every point without building the engine.  Returns the number kept, or -1 on a bad argument.
int64_t sm_oracle_random_sampler_mt19937(float rate, uint32_t seed, int64_t n, uint8_t* keep) {
  if (n < 0 || (n > 0 && !keep)) return -1;
  int64_t kept = 0;
  if (rate > 0.999) {
    for (int64_t j = 0; j < n; ++j) keep[j] = 1;
    return n;
  }
  std::mt19937 eng(seed);
  std::uniform_real_distribution<> distr(0., 1.);
  for (int64_t j = 0; j < n; ++j) {
    keep[j] = distr(eng) <= rate ? 1 : 0;
    kept += keep[j];
  }
  return kept;
}

}  // extern "C"
