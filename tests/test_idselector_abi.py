"""IDSelector construction and membership through the C ABI (no GPU): faiss_IDSelector_is_member must follow
the CPU's is_member (faiss/impl/IDSelector.{h,cpp}), restated in oracle/oracle_sel_np.py."""
import ctypes

import numpy as np
import pytest

import faiss_b200 as fb
from oracle import oracle_sel_np as osel


def to_fb(spec):
    kind = spec[0]
    if kind == "range":
        return fb.IDSelectorRange(spec[1], spec[2])
    if kind == "array":
        return fb.IDSelectorArray(spec[1])
    if kind == "batch":
        return fb.IDSelectorBatch(spec[1])
    if kind == "bitmap":
        return fb.IDSelectorBitmap(spec[1])
    if kind == "not":
        return fb.IDSelectorNot(to_fb(spec[1]))
    cls = {"and": fb.IDSelectorAnd, "or": fb.IDSelectorOr, "xor": fb.IDSelectorXOr}[kind]
    return cls(to_fb(spec[1]), to_fb(spec[2]))


PROBE = np.array(
    [-(2**63), -(2**40), -5, -1, 0, 1, 2, 3, 4, 7, 8, 9, 19, 20, 79, 80, 99, 100, 101, 799, 800, 801, 2**40, 2**63 - 1],
    dtype=np.int64,
)


@pytest.mark.parametrize("name", list(osel.reference_selectors(100)))
def test_reference_selectors_match_is_member(name):
    spec = osel.reference_selectors(100)[name]
    sel = to_fb(spec)
    ids = np.concatenate([PROBE, np.arange(-3, 110, dtype=np.int64)])
    want = osel.is_member(spec, ids)
    got = np.array([sel.is_member(int(i)) for i in ids])
    assert np.array_equal(got, want)


def test_negative_and_large_ids():
    ids = np.array([-7, 2**40 + 3, 5, -(2**62)], dtype=np.int64)
    sel = fb.IDSelectorBatch(ids)
    assert [sel.is_member(int(i)) for i in ids] == [True] * 4
    assert not sel.is_member(-6) and not sel.is_member(2**40 + 2)
    rng = fb.IDSelectorRange(-10, -2)
    assert rng.is_member(-10) and rng.is_member(-3) and not rng.is_member(-2) and not rng.is_member(0)


def test_bitmap_past_n_and_negative_ids():
    sel = fb.IDSelectorBitmap(np.array([0xFF, 0x01], dtype=np.uint8))
    assert all(sel.is_member(i) for i in range(9))
    assert not sel.is_member(9) and not sel.is_member(16) and not sel.is_member(10**12)
    # a negative id is a huge unsigned value: past any bitmap
    assert not sel.is_member(-1) and not sel.is_member(-(2**63))


def test_empty_range_and_empty_sets():
    assert not any(fb.IDSelectorRange(5, 5).is_member(i) for i in range(-2, 10))
    assert not any(fb.IDSelectorRange(9, 3).is_member(i) for i in range(-2, 12))
    assert not fb.IDSelectorArray([]).is_member(0)
    assert not fb.IDSelectorBatch(np.zeros(0, np.int64)).is_member(0)
    assert not fb.IDSelectorBitmap(np.zeros(0, np.uint8)).is_member(0)


def test_array_duplicates_select_by_membership():
    sel = fb.IDSelectorArray([3, 3, 3, 1000])
    assert sel.is_member(3) and sel.is_member(1000) and not sel.is_member(4)


def test_callback_and_combinators_keep_children():
    sel = fb.IDSelectorAnd(fb.IDSelectorCallback(lambda i: i % 2 == 0), fb.IDSelectorNot(fb.IDSelectorRange(0, 4)))
    want = [(i % 2 == 0) and not (0 <= i < 4) for i in range(-2, 9)]
    assert [sel.is_member(i) for i in range(-2, 9)] == want


def test_error_codes():
    lib = fb.lib
    out = ctypes.c_void_p()
    # null operands / inputs: FaissException -> -2, no handle written
    assert lib.faiss_IDSelectorNot_new(ctypes.byref(out), None) == -2
    assert b"null" in lib.faiss_get_last_error()
    assert lib.faiss_IDSelectorAnd_new(ctypes.byref(out), None, None) == -2
    assert lib.faiss_IDSelectorBatch_new(ctypes.byref(out), ctypes.c_size_t(3), None) == -2
    assert lib.faiss_IDSelectorBitmap_new(ctypes.byref(out), ctypes.c_size_t(3), None) == -2
    assert lib.faiss_b200_IDSelectorCallback_new(ctypes.byref(out), None, None) == -2
    assert lib.faiss_IDSelector_is_member(None, ctypes.c_int64(0)) == -1
    lib.faiss_IDSelector_free(None)  # no-op


def test_search_parameters_carry_the_selector():
    sel = fb.IDSelectorRange(0, 10)
    sp = fb.SearchParameters(sel=sel)
    assert sp.sel is sel
    ivf = fb.SearchParametersIVF(nprobe=7, sel=sel)
    assert ivf.sel is sel
    assert fb.SearchParametersIVF(nprobe=3).sel is None
