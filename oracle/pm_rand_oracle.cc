// glibc's rand() stream and libpointmatcher 1.3.1's RandomSamplingDataPointsFilter drawn from it, for the
// IcpUsingPointMatcher stand-in's rand reading sampler (sm_set_pm_reading_sampler).  The stream is glibc's own:
// rand() is random(), whose state is TYPE_3 (a 128-byte buffer); initstate_r / srandom_r / random_r run that
// generator on a private buffer, so no restatement of it is involved here.
#include <cstdint>
#include <cstdlib>
#include <cstring>

namespace {

// srand(seed), then `position` draws discarded
bool seeded_at(uint32_t seed, int64_t position, int32_t* state_words, random_data* buf) {
  memset(buf, 0, sizeof(*buf));
  if (initstate_r(seed, reinterpret_cast<char*>(state_words), 128, buf) != 0) return false;
  if (srandom_r(seed, buf) != 0) return false;
  int32_t r;
  for (int64_t i = 0; i < position; ++i) random_r(buf, &r);
  return true;
}

}  // namespace

extern "C" {

// draws position .. position + count - 1 of the rand() stream after srand(seed)
int sm_oracle_glibc_rand(uint32_t seed, int64_t position, int64_t count, int32_t* out) {
  if (position < 0 || count < 0 || (count > 0 && !out)) return -1;
  int32_t state[32];
  random_data buf;
  if (!seeded_at(seed, position, state, &buf)) return -1;
  for (int64_t i = 0; i < count; ++i) random_r(&buf, &out[i]);
  return 0;
}

// RandomSamplingDataPointsFilter::inPlaceFilter (libpointmatcher 1.3.1) over n columns with the stream at
// `position` after srand(seed): column i is kept iff (float)rand() / (float)RAND_MAX < prob, one draw per column.
// keep_n[i] = 0 / 1; returns the number kept, or -1 on a bad argument.
int64_t sm_oracle_pm_rand_mask(uint32_t seed, int64_t position, float prob, int64_t n, uint8_t* keep_n) {
  if (position < 0 || n < 0 || (n > 0 && !keep_n)) return -1;
  int32_t state[32];
  random_data buf;
  if (!seeded_at(seed, position, state, &buf)) return -1;
  int64_t kept = 0;
  for (int64_t i = 0; i < n; ++i) {
    int32_t r;
    random_r(&buf, &r);
    const float v = (float)r / (float)RAND_MAX;
    keep_n[i] = v < prob ? 1 : 0;
    kept += keep_n[i];
  }
  return kept;
}

}  // extern "C"
