"""The producer x consumer table of operand_states.py and its host models, without a
device: every pair is run or excluded for a stated reason, and the quirk models say
what the code they restate does."""
import numpy as np

import mxv_reference as ref
import operand_states as st
from support import Csr, csr


def test_every_pair_is_run_or_excluded_with_a_reason():
    pairs = set(st.ALL_PAIRS)
    assert len(pairs) == len(st.PRODUCERS)*len(st.CONSUMERS)
    assert set(st.RUN) | set(st.EXCLUDED) == pairs
    assert not set(st.RUN) & set(st.EXCLUDED)
    for pc, reason in st.EXCLUDED.items():
        assert reason in st.REASONS and st.REASONS[reason].strip(), pc
    # every reason is used, and no producer or consumer is excluded from everything
    assert set(st.EXCLUDED.values()) == set(st.REASONS)
    ran_p = {p for p, _ in st.RUN}
    ran_c = {c for _, c in st.RUN}
    assert ran_p == set(st.PRODUCERS)
    order_dependent = {"reduce_gt", "reduce_lt", "reduce_ne"}
    assert ran_c == set(st.CONSUMERS) - order_dependent


def test_the_table_holds_every_required_state_and_read():
    assert set(st.REQUIRED_PRODUCERS) <= set(st.PRODUCERS)
    for s in st.STATES:
        assert "dup_" + s in st.PRODUCERS and "swap_" + s in st.PRODUCERS
    for name in st.MONOID_NAMES:
        assert "reduce_" + name in st.CONSUMERS
    for c in ("extract_dense", "extract_sparse", "extract_into", "device_ptr", "bits",
              "ewise_add_self", "ewise_add_as_w", "ewise_mult_self", "assign_mask",
              "assign_mask_scmp", "gather", "scatter", "mxv_u_pull", "vxm_u_push",
              "mxv_mask_pull", "vxm_mask_push", "mxv_w_accum", "dense2sparse",
              "mis_candidates", "mis_self", "lgc_sweep"):
        assert c in st.CONSUMERS, c


def test_static_classes_name_producers():
    for group in (st.SPARSE_PRODUCERS, st.PATTERN_PRODUCERS, st.HUGE_PRODUCERS):
        assert group <= set(st.PRODUCERS)
    assert st.PATTERN_PRODUCERS <= st.SPARSE_PRODUCERS
    # the struct-only compactions, and only they, leave a pattern without values
    assert st.PATTERN_PRODUCERS == {p for p in st.PRODUCERS
                                    if p.startswith("dense2sparse") and p.endswith("so1")}


def test_the_operand_model():
    op = st.Operand(None, ind=[3, 9], val=[2, 0])
    assert op.sparse and "pattern" not in op.tags
    assert op.x.shape == (st.N,) and op.x[3] == 2 and op.x.sum() == 2
    op = st.Operand(None, ind=[3], val=None)
    assert "pattern" in op.tags and not op.x.any()
    op = st.Operand(None, np.full(st.N, st.FLT_MAX, np.float32))
    assert not op.sparse and "huge" in op.tags


def test_quirk_models():
    before = np.float32([5, 5, 5])
    assert np.array_equal(st.opreuse_sparse2dense(before), before)
    S = csr(3, 4, [0, 0, 1, 2], [0, 1, 2, 3], np.float32([1, 2, 3, 0]), np.float32)
    # plus-times from rows 0 and 2: row 2 holds only a 0 (dropped under a mask)
    f, fv = np.int32([0, 2]), np.float32([1, 5])
    ind, val = ref.push(1, S.ptr, S.ind, S.val, f, fv, 4)
    assert list(ind) == [0, 1, 3] and list(val) == [1, 2, 0]
    ind, val = st.masked_push(1, S, f, fv, 4, np.ones(4, np.float32))
    assert list(ind) == [0, 1] and list(val) == [1, 2]
    ind, val = st.struct_push(1, S, f, fv, 4)
    assert list(ind) == [0, 1, 3] and list(val) == [1, 1, 1]
    assert isinstance(S, Csr)


def test_mul_reduce_is_compared_only_where_every_order_agrees():
    assert st.mul_reduce_defined(np.float32([0, 1, -1, 2, 0.5]))
    assert not st.mul_reduce_defined(np.float32([3, 1]))
    assert not st.mul_reduce_defined(np.full(200, 2, np.float32))
    assert st.mul_reduce_defined(np.zeros(10, np.float32))


def test_expected_reduce_launches():
    dense = st.Operand(None, np.zeros(st.N, np.float32), tags=("counted", "zero_one"))
    assert st.reduce_launches(dense, 0) == 0
    assert st.reduce_launches(dense, 2) is None
    dup = st.Operand(None, np.zeros(st.N, np.float32), tags=("zero_one",))
    assert st.reduce_launches(dup, 0) == 1
    assert st.reduce_launches(st.Operand(None, np.zeros(st.N, np.float32)), 0) is None
    assert st.reduce_launches(st.Operand(None, ind=[1], val=[1]), 0) is None
