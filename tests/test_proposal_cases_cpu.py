"""CPU: the case builders of tests/proposal_cases.py really build what the GPU path tests rely on -- the dispatch
boundaries, borderline IoU pairs of every class, a column whose NMS is decided past scan word 16, images that trip the
decode kernel's structure gate, and ulp-apart score pairs."""
from fractions import Fraction

import numpy as np
import pytest

import proposal_cases as P
from oracle import postproc

F32 = np.float32


def test_dispatch_boundaries():
    assert P.dispatch(51, 20) == ("column-static", "bucketed")
    assert P.dispatch(52, 20) == ("column-optin", "bucketed")
    assert P.dispatch(116, 4) == ("column-optin", "bucketed")
    assert P.dispatch(117, 4) == ("generic-all", None)
    assert P.dispatch(8, 256) == ("column-static", "bucketed")
    assert P.dispatch(8, 257) == ("column-static", "gathered")
    assert P.dispatch(37, 56, feat_stride=8) == ("generic-all", None)
    assert P.dispatch(37, 56, feat_stride=32) == ("column-static", "bucketed")
    assert P.dispatch(62, 37, lib={"CTPN_COLUMN_GATHER": "1"}) == ("column-optin", "gathered")
    assert P.dispatch(62, 37, lib={"CTPN_GENERIC_NMS": "1"}) == ("generic-all", None)
    # the limits themselves: static shared memory ends between H = 51 and 52, the opt-in column kernel at 116 / 117
    assert P.column_smem_bytes(51) <= P.STATIC_SMEM < P.column_smem_bytes(52)
    assert P.column_smem_bytes(116) <= P.OPTIN_SMEM < P.column_smem_bytes(117)
    assert (116 * 10 + 63) // 64 == 19                     # scan words of the tallest column map


def _check_pair_classes(a, b, thresh, classes):
    T = Fraction(float(F32(thresh)))
    inter, u, q = P.iou_terms(a, b)
    np.testing.assert_array_equal(P.postproc.iou_row(a, b[None]), [q])       # same float32 IoU as the oracle
    fi, fu = Fraction(float(inter)), Fraction(float(u))
    band = abs(fi - T * fu) <= Fraction(1, 2 ** 20) * max(fi, fu)
    if "eq" in classes:
        assert Fraction(float(q)) == T
    if "eq_above" in classes:
        assert fi / fu > T and Fraction(float(q)) == T
    if "exact" in classes:
        assert fi / fu == T
    if "up" in classes:
        assert q == np.nextafter(F32(thresh), F32(np.inf))
    if "down" in classes:
        assert q == np.nextafter(F32(thresh), F32(-np.inf))
    if "band_above" in classes:
        assert band and fi / fu > T
    if "band_below" in classes:
        assert band and fi / fu < T


@pytest.mark.parametrize("thresh", [0.7, 0.5])
def test_column_pairs_cover_every_class(thresh):
    pairs = P.column_pairs(thresh)
    for cl in P.required_classes(thresh):
        assert sum(cl in p[-1] for p in pairs) >= 3, cl
    cls, bbox, info, idx = P.column_pair_heads(pairs)
    boxes, _, valid = P.decoded(cls, bbox, info)
    assert valid.sum() == 2 * len(pairs) and all(valid[i] and valid[j] for i, j in idx)   # only the pairs are valid
    for (i, j), p in zip(idx, pairs):
        _check_pair_classes(boxes[i], boxes[j], thresh, p[-1])
    assert not P.gate_triggers(cls, bbox, info, nms_thresh=thresh)                       # the column path takes it
    assert P.dispatch(*cls.shape[1:3]) == ("column-static", "bucketed")
    # the oracle keeps both boxes of a pair exactly when the float32 IoU is not above T
    _, _, kept = postproc.proposal_layer(cls, bbox, info, nms_thresh=thresh, return_index=True)
    for (i, j), p in zip(idx, pairs):
        assert i in kept and (j in kept) == (P.iou_terms(boxes[i], boxes[j])[2] <= F32(thresh))
    if F32(thresh) == F32(0.7):
        assert any("eq_above" in p[-1] and idx[k][1] in kept for k, p in enumerate(pairs))


@pytest.mark.parametrize("thresh", [0.7, 0.5, 0.3, 0.2])
def test_generic_pairs_cover_every_class(thresh):
    pairs = P.generic_pairs(thresh)
    for cl in P.required_classes(thresh, integer_boxes=True):
        assert sum(cl in p[-1] for p in pairs) >= 4, cl
    for wa, wb, ov, cl in pairs:
        _check_pair_classes(*P.generic_pair_boxes(wa, wb, ov), thresh, cl)
    dets = P.generic_pair_dets(pairs, 129, lead=1)
    assert (np.diff(dets[:, 4]) < 0).all()
    # a pair straddles the first block edge: positions 63 (A) and 64 (B)
    assert dets[63, 1] == dets[64, 1] and P.iou_terms(dets[63], dets[64])[0] > 0


def test_h116_column_is_decided_past_word_16():
    cls, bbox = P.random_heads(116, 1, 116, 4)
    count, suppressed = P.column_census(cls, bbox, np.array([[116 * 16, 64, 1.0]], F32))
    assert count.max() > 1024
    assert any(pos >= 1024 for col in suppressed for pos in col)


def test_gate_cases_trip_the_structure_check():
    cls, bbox, info = P.mixed_batch()
    assert P.gate_triggers(cls[0:1], bbox[0:1], info[0]) == set()
    assert P.gate_triggers(cls[1:2], bbox[1:2], info[1]) == {"x1", "width"}
    assert P.gate_triggers(cls[2:3], bbox[2:3], info[2]) == {"width"}
    for b in range(3):
        assert "width" in P.gate_triggers(cls[b:b + 1], bbox[b:b + 1], info[b], nms_thresh=0.03)


def test_ulp_pairs_are_present_in_both_parities():
    cls, bbox, pairs = P.ulp_pair_heads(75, 100)
    fg = cls[0, ..., 1::2].reshape(-1)
    lo, hi = fg[pairs[:, 0]], fg[pairs[:, 1]]
    assert (hi == np.nextafter(lo, F32(np.inf))).all() and (pairs[:, 1] > pairs[:, 0]).all()
    parity = lo.view(np.uint32) & 1
    assert (parity == 0).sum() >= 10 and (parity == 1).sum() >= 10
    _, _, valid = P.decoded(cls, bbox, np.array([[1200, 1600, 1.0]], F32))
    assert valid[pairs.ravel()].all()
    # everything else is on the 1/64 grid: large tie groups
    assert len(np.unique(fg)) <= 63 + 2 * len(pairs)


def test_min_size_boundary_case():
    """dh = 0: anchor 0's box is exactly 13 rows high (+1 convention), so RPN_MIN_SIZE = 13 keeps it (>=) and 13.5
    drops it; the widths (17) pass either way."""
    cls, bbox = P.exact_heads(6, 5)
    cls[..., 1::2] = F32(0.5)
    for ms, want in ((13, 30), (13.5, 0)):
        _, _, valid = P.decoded(cls, bbox, np.array([[96, 80, 1.0]], F32), min_size=ms)
        assert valid.reshape(-1, 10)[:, 0].sum() == want
