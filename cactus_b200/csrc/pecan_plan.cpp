// pecan_plan.cpp -- see pecan_plan.h. Host only (also compiled into tests/hosttest).
#include "pecan_plan.h"
#include <math.h>
#include <algorithm>

namespace barb200 {
namespace pecan {

std::string check_params(const PlanParams &P) {
    // the prerequisites getPosteriorProbsWithBanding asserts, pairwiseAligner.c:771-775
    if (P.tb_diags < 1) return "traceBackDiagonals must be >= 1";
    if (P.expansion < 0 || P.expansion % 2 != 0) return "diagonalExpansion must be even and >= 0";
    if (P.min_diags < 2) return "minDiagsBetweenTraceBack must be >= 2";
    if (P.tb_diags + 1 >= P.min_diags) return "traceBackDiagonals + 1 must be < minDiagsBetweenTraceBack";
    if (!(P.threshold >= 0.0 && P.threshold <= 1.0)) return "threshold must be in [0, 1]";
    if (P.split_bigger < 1) return "splitMatrixBiggerThanThis must be >= 1";
    return "";
}

std::string check_anchors(const int64_t *a, int64_t n, int64_t lx, int64_t ly) {
    int64_t px = -1, py = -1;                      // band_construct's assertions, pairwiseAligner.c:222-228
    for (int64_t i = 0; i < n; ++i) {
        const int64_t x = a[2 * i], y = a[2 * i + 1];
        if (x <= px || y <= py || x >= lx || y >= ly || x < 0 || y < 0) return "anchor pairs must be strictly increasing in x and y and inside the sequences";
        px = x; py = y;
    }
    return "";
}

namespace {
struct Split { int64_t x1, y1, x2, y2; };

// getSplitPointsP, pairwiseAligner.c:1241-1263
bool split_p(int64_t *x1, int64_t *y1, int64_t x2, int64_t y2, int64_t x3, int64_t y3, std::vector<Split> &sp, int64_t bigger, bool skip) {
    const int64_t lX2 = x3 - x2, lY2 = y3 - y2;
    if (lX2 * lY2 > bigger) {
        const int64_t max_len = (int64_t)sqrt((double)bigger);
        const int64_t hX = lX2 / 2 > max_len ? max_len : lX2 / 2, hY = lY2 / 2 > max_len ? max_len : lY2 / 2;
        if (!skip) sp.push_back(Split{*x1, *y1, x2 + hX, y2 + hY});
        *x1 = x3 - hX; *y1 = y3 - hY;
        return true;
    }
    return false;
}
}  // namespace

void split_pair(const PlanParams &P, int64_t pair, int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor,
                bool ragged_left, bool ragged_right, std::vector<SubJob> &out) {
    std::vector<Split> sp;
    int64_t x1 = 0, y1 = 0, x2 = 0, y2 = 0;
    for (int64_t i = 0; i < n_anchor; ++i) {       // getSplitPoints, pairwiseAligner.c:1265-1292
        const int64_t x3 = anchors[2 * i], y3 = anchors[2 * i + 1];
        split_p(&x1, &y1, x2, y2, x3, y3, sp, P.split_bigger, ragged_left && i == 0);
        x2 = x3 + 1; y2 = y3 + 1;
    }
    const bool last_split = split_p(&x1, &y1, x2, y2, lx, ly, sp, P.split_bigger, ragged_left && n_anchor == 0);
    if (!last_split || !ragged_right) sp.push_back(Split{x1, y1, lx, ly});
    int64_t j = 0;
    for (size_t i = 0; i < sp.size(); ++i) {       // pairwiseAligner.c:1318-1350
        SubJob s;
        s.pair = pair; s.x1 = sp[i].x1; s.y1 = sp[i].y1;
        s.lx = (int)(sp[i].x2 - sp[i].x1); s.ly = (int)(sp[i].y2 - sp[i].y1);
        while (j < n_anchor) {
            const int64_t x = anchors[2 * j], y = anchors[2 * j + 1];
            if (x + y >= sp[i].x2 + sp[i].y2) break;
            s.anchors.push_back(x - sp[i].x1); s.anchors.push_back(y - sp[i].y1);
            ++j;
        }
        s.ragged = ((ragged_left || i > 0) ? 1 : 0) | ((ragged_right || i + 1 < sp.size()) ? 2 : 0);
        out.push_back(std::move(s));
    }
}

namespace {
inline int64_t avoid_off_by_one(int64_t xay, int64_t xmy) { return xmy + ((xay + xmy) & 1); }   // parity of a two's complement sum
inline int64_t bound(int64_t z, int64_t l) { return z < 0 ? 0 : (z > l ? l : z); }
// diagonal_getXCoordinate / YCoordinate use C division (truncation toward zero) on values that are even by construction
// everywhere except in band_construct's xL..yU, where the reference relies on the same truncation: keep `/ 2`.
}  // namespace

std::string plan_subjob(const PlanParams &P, SubJob &s) {
    const int64_t lX = s.lx, lY = s.ly, D = lX + lY, n_anchor = (int64_t)s.anchors.size() / 2;
    s.bandL.assign(D + 1, 0); s.coff.assign(D + 2, 0);
    int64_t ai = 0, xay = 0, pxay = 0, pxmy = 0, nxay = 0, nxmy = 0, xL = 0, yL = 0, xU = 0, yU = 0, cells = 0;
    int max_w = 0;
    while (xay <= D) {                              // band_construct, pairwiseAligner.c:193-244
        int64_t l = avoid_off_by_one(xay, xL - yL), r = avoid_off_by_one(xay, xU - yU), i;
        // (xay + l), (xay - l), ... are even here, so the reference's "/ 2" is an exact shift
        i = (xay + l) >> 1; if (i < xL) l += 2 * (xL - i);           // band_setCurrentDiagonal, :114-132
        i = (xay - l) >> 1; if (yL < i) l += 2 * (i - yL);
        i = (xay + r) >> 1; if (xU < i) r -= 2 * (i - xU);
        i = (xay - r) >> 1; if (i < yU) r -= 2 * (yU - i);
        if (l > r || ((xay + l) & 1) || ((xay + r) & 1)) return "invalid band diagonal (the reference throws PAIRWISE_ALIGNMENT_EXCEPTION here)";
        const int64_t w = ((r - l) >> 1) + 1;
        s.bandL[xay] = (int)l; s.coff[xay] = (int)cells;
        cells += w; max_w = std::max<int64_t>(max_w, w);
        if (cells > (int64_t)400 * 1000 * 1000) return "pair-HMM job larger than 4e8 banded cells";
        if (nxay == xay++) {
            pxay = nxay; pxmy = nxmy;
            int64_t x = lX, y = lY;
            if (ai < n_anchor) { x = s.anchors[2 * ai] + 1; y = s.anchors[2 * ai + 1] + 1; ++ai; }
            nxay = x + y; nxmy = x - y;
            xL = bound((pxay + (pxmy - P.expansion)) / 2, lX);
            yL = bound((nxay - (nxmy - P.expansion)) / 2, lY);
            xU = bound((nxay + (nxmy + P.expansion)) / 2, lX);
            yU = bound((pxay - (pxmy + P.expansion)) / 2, lY);
        }
    }
    s.coff[D + 1] = (int)cells;
    s.cells = cells; s.max_w = max_w;
    {   // where the band's cells sit on the ring coordinate a = (xmy + parity) / 2 + ly (pecan_cta.cuh): their mean
        double acc = 0;
        for (int64_t d = 0; d <= D; ++d) {
            const int64_t w = s.coff[d + 1] - s.coff[d], a0 = ((s.bandL[d] + (d & 1)) >> 1) + lY;
            acc += (double)w * (double)a0 + 0.5 * (double)w * (double)(w - 1);
        }
        s.ring_center = (int)(acc / (double)std::max<int64_t>(cells, 1));
    }
    // schedule (pairwiseAligner.c:798-803, 817, 840-848): traceback points only depend on the band geometry
    std::vector<uint8_t> mark((size_t)D + 1, 0);
    s.tb_from.clear();
    struct Tb { int64_t d, to; };
    std::vector<Tb> tbs;
    int64_t tb_to = 0;
    for (int64_t d = 1; d <= D; ++d) {
        const int64_t w = s.coff[d + 1] - s.coff[d];
        const bool at_end = d == D, tb_point = d >= tb_to + P.min_diags && w <= P.expansion * 2 + 1;
        if (!(at_end || tb_point)) continue;
        const int64_t tb_from = d - (at_end ? 0 : P.tb_diags + 1);
        int64_t c = 0;
        for (int64_t t = tb_from; t > tb_to; --t, ++c)
            if (c % 10 == 0) { mark[t] = 1; mark[t - 1] = 1; }
        if (!at_end) { mark[d] = 1; mark[d - 1] = 1; }
        tbs.push_back(Tb{d, tb_to});
        s.tb_from.push_back((int)tb_from);
        tb_to = tb_from;
    }
    s.foff.assign(D + 2, 0);
    int64_t fc = 0;
    for (int64_t d = 0; d <= D; ++d) { s.foff[d] = (int)fc; if (mark[d]) fc += s.coff[d + 1] - s.coff[d]; }
    s.foff[D + 1] = (int)fc;
    int64_t span = 1, span_full = 1;
    for (const Tb &tb : tbs) {
        span = std::max<int64_t>(span, s.coff[tb.d + 1] - s.coff[tb.to]);
        span_full = std::max<int64_t>(span_full, s.foff[tb.d + 1] - s.foff[tb.to]);
    }
    s.span_cells = span; s.span_full_cells = span_full;
    return "";
}

std::vector<std::vector<int64_t>> deal_pairs(const std::vector<int64_t> &cost, int ndev) {
    const int64_t n = (int64_t)cost.size();
    ndev = std::max(ndev, 1);
    std::vector<std::vector<int64_t>> share(ndev);
    std::vector<int64_t> idx(n);
    for (int64_t i = 0; i < n; ++i) idx[i] = i;
    if (ndev == 1) { share[0] = std::move(idx); return share; }
    std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) { return cost[a] > cost[b]; });
    std::vector<int64_t> load(ndev, 0);
    for (int64_t i : idx) { const int d = (int)(std::min_element(load.begin(), load.end()) - load.begin()); share[d].push_back(i); load[d] += cost[i]; }
    for (auto &s : share) std::sort(s.begin(), s.end());
    return share;
}

}  // namespace pecan
}  // namespace barb200
