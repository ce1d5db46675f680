// gt_keys.cpp -- TEST-ONLY: the number of minimizer keys the product's guide tree (cactus_b200/csrc/guide_tree.cuh: cta_guide_tree)
// appends for one job, the count the device compares with its key capacity (JOB_ERR_GT_CAP). The key array is sized at the
// worst case of slot_plan.h's GtNeeds, so the count is never cut short. Compiled by tests/test_repeats_cpu.py.
#include <vector>
#include "../../cactus_b200/csrc/slot_plan.h"

using namespace barb200;

// slot memory as the device has it: 256-byte aligned blocks
struct alignas(256) GkBlock { uint8_t b[256]; };

// Returns n_keys after the sketch, or -1 if cta_guide_tree reported a full key array (it cannot at the worst case).
extern "C" long long gt_keys_count(int k, int w, int progressive, int n_seq, const int *lens, const uint8_t *flat) {
    std::vector<const uint8_t *> seqs(n_seq);
    int64_t sum = 0;
    for (int i = 0; i < n_seq; ++i) { seqs[i] = flat + sum; sum += lens[i]; }
    GtNeeds need;
    need.add_job(progressive, n_seq, sum, w, 1.0, true);
    const GtLayout Y = plan_gt_scratch(need);
    std::vector<GkBlock> scratch((size_t)Y.slot_bytes / sizeof(GkBlock));
    std::vector<uint64_t> tile(2048);
    std::vector<int> order(n_seq);
    int n_keys = 0; double wsv[33]; long long wsi[33];
    GtScratch G = gt_views(Y, scratch.data()->b);
    G.n_keys = &n_keys; G.tile = tile.data(); G.tile_cap = (int)tile.size();
    const GuideTreeParams GP{k, w};
    if (cta_guide_tree(GP, progressive, n_seq, [&](int i) { return seqs[i]; }, lens, order.data(), G, wsv, wsi, 64) != 0) return -1;
    return n_keys;
}
