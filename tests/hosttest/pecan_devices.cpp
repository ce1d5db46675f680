// pecan_devices.cpp -- TEST-ONLY host build of the deal of a cPecan batch over devices (cactus_b200/csrc/pecan_plan.cpp:
// deal_pairs) behind a C symbol. tests/test_pecan_devices_cpu.py compiles this file with pecan_plan.cpp into a temporary
// directory; never shipped, never loaded by cactus_b200.
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "../../cactus_b200/csrc/pecan_plan.h"

// n pairs of cost[n] over ndev devices -> counts[ndev] and every device's share back to back in pairs[n]
extern "C" void hosttest_pecan_deal_pairs(int64_t n, const int64_t *cost, int ndev, int64_t *counts, int64_t *pairs) {
    for (const std::vector<int64_t> &s : barb200::pecan::deal_pairs(std::vector<int64_t>(cost, cost + n), ndev)) {
        *counts++ = (int64_t)s.size(); pairs = std::copy(s.begin(), s.end(), pairs);
    }
}
