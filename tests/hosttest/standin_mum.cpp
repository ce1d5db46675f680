// standin_mum.cpp -- TEST-ONLY: the MUM anchor entries of the C ABI (barb200_mum_params_default, barb200_pecan_anchor_pairs_batch)
// for the stand-in device (standin_device.cpp), every pair through the host build of K5 (mum_host.cpp). Linked only into
// libbarb200_standin_mum.so (mum.mk), under which oracle/mum.mk runs the real pecan shim in cPecan bar().
#include <stdlib.h>
#include <string>
#include "../../cactus_b200/csrc/host_api.h"

extern "C" int64_t hosttest_mum_anchor_pairs(const char *sx, int64_t lx, const char *sy, int64_t ly, int64_t k, int64_t u, int64_t bigger,
                                             int recursive, uint64_t tie_seed, int64_t **out);

extern "C" void barb200_mum_params_default(barb200_mum_params *p) {
    p->k = 50; p->u = 1; p->anchor_matrix_bigger_than_this = (int64_t)500 * 500; p->recursive_mums = 1;
}

extern "C" int barb200_pecan_anchor_pairs_batch(barb200_ctx *ctx, const barb200_mum_params *p, int64_t n_pairs, const char *const *sx, const int64_t *lx,
                                                const char *const *sy, const int64_t *ly, int64_t **anchors_out, int64_t *n_anchor_out) {
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int64_t n = hosttest_mum_anchor_pairs(sx[i], lx[i], sy[i], ly[i], p->k, p->u, p->anchor_matrix_bigger_than_this, p->recursive_mums, 0,
                                                    &anchors_out[i]);
        if (n < 0) {
            for (int64_t j = 0; j < i; ++j) { free(anchors_out[j]); anchors_out[j] = nullptr; }
            barb200::set_error(ctx, "stand-in device: MUM anchor parameters or bytes rejected");
            return BARB200_EINVAL;
        }
        n_anchor_out[i] = n;
    }
    return BARB200_OK;
}
