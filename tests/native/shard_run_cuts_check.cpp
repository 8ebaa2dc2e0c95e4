// The shard-run cut planner of sharded input over a group (shard_range.hpp shard_run_cuts): `shard_run_cuts_check N size...`
// prints the N + 1 cuts (tests/test_sharded_group.py checks them against a brute-force search).
#include <cstdio>
#include <cstdlib>

#include "coverm_b200.h"
#include "shard_range.hpp"

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::vector<uint64_t> sizes;
  for (int i = 2; i < argc; ++i) sizes.push_back(strtoull(argv[i], nullptr, 10));
  for (uint32_t c : cmbh::shard_run_cuts(sizes, atoi(argv[1]))) printf("%u ", c);
  printf("\n");
  return 0;
}
