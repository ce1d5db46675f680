"""The memory layout of a POA slot and of a guide-tree scratch slot (cactus_b200/csrc/slot_plan.h), CPU only. The stage plan, the
kernels and the CPU build of the graph code all take their arrays from it: every array must lie inside its slot, apart from
every other, 16-byte aligned, and a slot must be a multiple of 256 bytes. The capacities come from the layout; each array's
size is worked out here from the element type and count that poa_types.h (Graph, RowTables, DpState) and guide_tree.cuh
(GtScratch) give, not read back from the code under test."""
import ctypes as C

import pytest

import _reflib as R

WB, WF = 1000, 0.1                      # Cactus' band (cactus_progressive_config.xml)
MINIMIZER_W = 5                         # partialOrderAlignmentMinimizerW default
KS = (1, 2, 64, 65, 90)                 # 65: two 64-bit words per read-id set
LENS = (1, 511, 2047, 10000, 16383)

SLOT_CAPS = ("slot_bytes", "node_cap", "in_pool", "out_pool", "W", "cigar_cap", "fc_cap", "plane_cap")
SLOT_ARRAYS = ("base", "aln_n", "aln_id", "in_off", "in_n", "in_cap", "out_off", "out_n", "out_cap",
               "in_id", "in_w", "out_id", "out_w", "out_rid",
               "index_to_node", "node_to_index", "remain", "msa_rank", "tmp0", "tmp1",
               "row_rec", "pre_row", "row_off", "row_info", "cigar", "fc")
GT_CAPS = ("slot_bytes", "key_cap", "base_cap", "seq_cap")
GT_ARRAYS = ("keys", "gx", "hit", "jac", "score")


def _lib():
    lib = R._load(R.build_hosttest())
    lib.hosttest_slot_layout.restype = None
    lib.hosttest_slot_layout.argtypes = [C.c_int64] * 4 + [C.POINTER(C.c_int64)]
    lib.hosttest_gt_layout.restype = None
    lib.hosttest_gt_layout.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_double, C.c_int, C.POINTER(C.c_int64)]
    lib.hosttest_plane_ints_for_job.restype = C.c_int64
    lib.hosttest_plane_ints_for_job.argtypes = [C.c_int, C.c_double, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int]
    return lib


def slot_layout(lib, K, L):
    planes = lib.hosttest_plane_ints_for_job(WB, WF, K, K * L, L, 1.0, 0)
    out = (C.c_int64 * (len(SLOT_CAPS) + len(SLOT_ARRAYS)))()
    lib.hosttest_slot_layout(K, K * L, L, planes, out)
    v = list(out)
    return dict(zip(SLOT_CAPS, v)), dict(zip(SLOT_ARRAYS, v[len(SLOT_CAPS):])), planes


def slot_sizes(c):
    N, I, O, W = c["node_cap"], c["in_pool"], c["out_pool"], c["W"]
    return {
        "base": 1 * N, "aln_n": 1 * N,                          # uint8_t [node_cap]
        "aln_id": 4 * N * 4,                                    # int [node_cap * 4]
        "in_off": 4 * N, "in_n": 4 * N, "in_cap": 4 * N,        # int [node_cap]
        "out_off": 4 * N, "out_n": 4 * N, "out_cap": 4 * N,
        "in_id": 4 * I, "in_w": 4 * I,                          # int [in_pool]
        "out_id": 4 * O, "out_w": 4 * O,                        # int [out_pool]
        "out_rid": 8 * O * W,                                   # uint64_t [out_pool * W]
        "index_to_node": 4 * N, "node_to_index": 4 * N, "remain": 4 * N, "msa_rank": 4 * N, "tmp0": 4 * N, "tmp1": 4 * N,
        "row_rec": 16 * N,                                      # RowRec (4 ints) [node_cap]
        "pre_row": 4 * I,                                       # int [in_pool]
        "row_off": 8 * N,                                       # int64_t [node_cap]
        "row_info": 16 * N,                                     # RowInfo (4 ints) [node_cap]
        "cigar": 8 * c["cigar_cap"],                            # uint64_t [cigar_cap]
        "fc": 4 * 2 * c["fc_cap"],                              # int [2 * fc_cap]
    }


def gt_sizes(c):
    K = c["seq_cap"]
    return {
        "keys": 8 * c["key_cap"],                               # uint64_t [key_cap]
        "gx": 8 * c["base_cap"],                                # uint64_t [bases of the job]
        "hit": 4 * (K * (K + 1) // 2),                          # int [K (K + 1) / 2]
        "jac": 8 * (K * (K - 1) // 2),                          # double [K (K - 1) / 2]
        "score": 8 * K,                                         # double [K]
    }


def check_packing(slot_bytes, offsets, sizes):
    assert slot_bytes % 256 == 0
    for name, o in offsets.items():
        assert o % 16 == 0, name
        assert 0 <= o and o + sizes[name] <= slot_bytes, name
    ranges = sorted((offsets[n], offsets[n] + sizes[n], n) for n in offsets if sizes[n] > 0)
    for (_, end, a), (start, _, b) in zip(ranges, ranges[1:]):
        assert end <= start, (a, b)


@pytest.mark.parametrize("L", LENS)
@pytest.mark.parametrize("K", KS)
def test_slot_arrays_are_packed_inside_the_slot(K, L):
    caps, offs, planes = slot_layout(_lib(), K, L)
    check_packing(caps["slot_bytes"], offs, slot_sizes(caps))
    # the capacities hold the job: every base a node besides source and sink, a read-id bit per read, a column per query base
    assert caps["node_cap"] >= K * L + 2 and 64 * caps["W"] >= K and caps["fc_cap"] >= L + 1
    assert caps["plane_cap"] >= planes and caps["plane_cap"] % 8 == 0


@pytest.mark.parametrize("worst_case", [False, True])
@pytest.mark.parametrize("L", LENS)
@pytest.mark.parametrize("K", KS)
def test_guide_tree_arrays_are_packed_inside_the_scratch(K, L, worst_case):
    out = (C.c_int64 * (len(GT_CAPS) + len(GT_ARRAYS)))()
    _lib().hosttest_gt_layout(1, K, K * L, MINIMIZER_W, 1.0, int(worst_case), out)
    v = list(out)
    caps, offs = dict(zip(GT_CAPS, v)), dict(zip(GT_ARRAYS, v[len(GT_CAPS):]))
    check_packing(caps["slot_bytes"], offs, gt_sizes(caps))
    kc = caps["key_cap"]
    assert kc >= 64 and kc & (kc - 1) == 0                    # the sort pads the keys to a power of two
    if K > 2:                                                   # only these jobs build a guide tree
        assert caps["base_cap"] >= K * L and caps["seq_cap"] >= K
        if worst_case:
            assert kc >= 2 * MINIMIZER_W * K * L + K
