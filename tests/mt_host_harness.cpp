// mt_host_harness.cpp — std::mt19937 (the engine boost::mt19937 is) for tests/test_floor_host.py: the first n outputs of the
// generator seeded with `seed`, the sequence RandomSampleConsensus's sample draws start from on every call.
#include <cstdint>
#include <random>

extern "C" void mt19937_outputs(uint32_t seed, uint32_t* out, int n) {
  std::mt19937 g(seed);
  for (int i = 0; i < n; i++) out[i] = (uint32_t)g();
}
