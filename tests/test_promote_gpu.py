"""GPU: the bf16x3p arithmetic -- three bf16 planes with the wgmma main accumulator promoted to round-to-nearest float32
at every pipeline step (CTPN_F_PROMOTE, CTPN_ARITH_BF16X3P).

Kernel cases run ctpn_conv3x3 with and without the flag on the same inputs in one process (tests/promote_checks.py, a
subprocess per case so that a faulting kernel fails one test instead of the session) against float64 on the exact operand values the planes carry.  Network cases hold the mode to the float64
oracle, to the float32 oracle's proposals, and to bit-exact batching."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import net_cpu, postproc, synth
from test_conv_gpu import DBG
from test_net_gpu import TAPS, _match_rois, rel_err, rows_matched

pytestmark = pytest.mark.gpu
RELU, POOL, F32 = 1, 2, 4


HERE = os.path.dirname(os.path.abspath(__file__))


def promote_check(B, H, W, cin, cout, taps, flags, nonneg=0, env=None, timeout=300):
    args = dict(B=B, H=H, W=W, cin=cin, cout=cout, taps=taps, flags=flags, nonneg=nonneg)
    cmd = [sys.executable, os.path.join(HERE, "promote_checks.py")] + ["--%s=%d" % kv for kv in args.items()]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(cmd[2:]), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


# (B, H, W, cin, cout, taps, flags, env)
LONG_K = [
    (1, 37, 56, 512, 512, 9, RELU, None),                         # K = 4608, plane output
    (1, 37, 56, 512, 512, 9, RELU | F32, None),                   # K = 4608, float32 output
    (1, 37, 56, 512, 512, 9, RELU | F32, dict(DBG, CTPN_TC_MCAST="0")),   # single-CTA variant (BN = 64 when promoted)
    (1, 37, 56, 512, 512, 9, RELU | F32, dict(DBG, CTPN_TC_BN="64")),
]


@pytest.mark.parametrize("case", LONG_K, ids=["planes", "f32", "single_cta", "bn64"])
def test_promoted_long_k_error_is_a_quarter_of_unpromoted(case):
    *shape, env = case
    res = promote_check(*shape, env=env)
    plain, prom = res["plain"]["max_err"], res["promoted"]["max_err"]
    print("K=%d max|err| plain %.3e promoted %.3e (%.1fx)" % (res["K"], plain, prom, plain / max(prom, 1e-30)))
    assert prom <= 0.25 * plain                 # H100: 1/15.7
    assert prom <= 1e-6 * res["scale"]          # H100: 3.7e-7


OTHER = [
    (1, 1, 2072, 512, 1024, 1, F32),          # the BiLSTM x-projection GEMM of one 600x900 image (taps = 1)
    (3, 75, 112, 64, 64, 9, RELU | POOL),     # fused 2x2 max-pool, odd height (75 -> 37)
    (1, 150, 225, 64, 128, 9, RELU),          # many tiles per CTA: pipeline phase wrap-around
    (1, 8, 16, 128, 128, 9, RELU | F32),      # one pixel tile: the single-CTA kernel of the product library
]


@pytest.mark.parametrize("case", OTHER, ids=lambda c: "B%d_%dx%d_c%d-%d_t%d_f%d" % c)
def test_promoted_kernel_against_float64(case):
    res = promote_check(*case)
    # H100: promoted 1.6-2.0e-7 relative to max|y|, 4.3-8.5x under the unpromoted error
    assert res["promoted"]["max_err"] <= 1e-6 * res["scale"]
    assert res["promoted"]["max_err"] <= 0.5 * res["plain"]["max_err"]


def test_promotion_removes_the_truncation_bias():
    """Every product positive (K = 4608): the unpromoted kernel's truncating adds pull the sum down, which shows as a negative
    mean signed error; promotion leaves at most 1/8 of that bias."""
    res = promote_check(1, 37, 56, 512, 512, 9, F32, nonneg=1)
    plain, prom = res["plain"]["mean_err"], res["promoted"]["mean_err"]
    print("mean signed error: plain %.3e promoted %.3e (scale %.3e)" % (plain, prom, res["scale"]))
    assert plain < 0
    assert abs(prom) <= abs(plain) / 8          # H100: -2.29e-4 -> -1.2e-6


def test_promote_interval_switch_still_beats_unpromoted():
    """CTPN_TC_PROMOTE=4 (test library): main chains of 4 steps, still well under the unpromoted error."""
    res = promote_check(1, 37, 56, 512, 512, 9, RELU | F32, env=dict(DBG, CTPN_TC_PROMOTE="4"))
    assert res["promoted"]["max_err"] <= 0.25 * res["plain"]["max_err"]     # H100: 1/15


# ---- network ----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


def test_layerwise_against_float64_oracle(weights):
    from ctpn_b200 import Engine
    im = synth.make_image(7, 96, 160)
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, weights, dtype=torch.float64, taps=TAPS)
    eng = Engine(weights, mode="bf16x3p", keep_activations=True)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    torch.cuda.synchronize()
    worst = {name: rel_err(eng.tap(name).cpu().numpy().reshape(ref[name].shape), ref[name]) for name in TAPS}
    worst["rpn_cls_score"] = rel_err(cls.cpu().numpy(), ref["rpn_cls_score"])
    worst["rpn_bbox_pred"] = rel_err(bbox.cpu().numpy(), ref["rpn_bbox_pred"])
    print({k: "%.2e" % v for k, v in worst.items()})
    assert max(worst.values()) < 2e-5, worst    # H100: 3.5e-6 (lstm_out), every other tap <= 8e-7


def test_head_logits_600x900_against_float64_oracle(weights):
    from ctpn_b200 import Engine
    im = synth.make_image(11)
    blob, _ = net_cpu.image_blob(im)
    ref = net_cpu.forward(blob, weights, dtype=torch.float64)
    cls, bbox = Engine(weights, mode="bf16x3p").forward_heads(torch.from_numpy(im[None]).cuda())
    d_cls = float(np.abs(cls.cpu().numpy() - ref["rpn_cls_score"]).max())
    d_box = float(np.abs(bbox.cpu().numpy() - ref["rpn_bbox_pred"]).max())
    print("bf16x3p seed 11 head max|diff| vs float64: cls %.2e bbox %.2e" % (d_cls, d_box))
    assert d_cls < 3e-5 and d_box < 1e-5        # H100: 7.8e-6 / 8.4e-7 (bf16x3: 2.1e-4 / 2.5e-5)


def test_end_to_end_600x900_against_oracle(weights):
    """The checks of test_net_gpu.test_end_to_end_600x900_against_oracle for the promoted mode; all 1000 rows."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x3p")
    im = synth.make_image(0)
    blob, scale = net_cpu.image_blob(im)
    assert scale == 1.0
    ref = net_cpu.forward(blob, weights)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    cls_h, bbox_h = cls.cpu().numpy(), bbox.cpu().numpy()
    d_cls, d_box = np.abs(cls_h - ref["rpn_cls_score"]).max(), np.abs(bbox_h - ref["rpn_bbox_pred"]).max()
    print("bf16x3p head max|diff| vs float32 oracle: cls %.2e bbox %.2e" % (d_cls, d_box))
    assert d_cls < 1e-4 and d_box < 1.5e-5      # H100: 4.3e-5 / 4.1e-6, mostly the float32 oracle's own rounding
    info = np.array([[600, 900, 1.0]], np.float32)
    rois, index, count = eng.proposals(cls, bbox, torch.from_numpy(info), cls_is_logit=True)
    n = int(count[0])
    assert n == 1000
    got, got_idx = rois[0, :n].cpu().numpy(), index[0, :n].cpu().numpy()
    l = cls_h.reshape(-1, 2).astype(np.float64)
    e = np.exp(l - l.max(1, keepdims=True))
    prob = (e / e.sum(1, keepdims=True)).astype(np.float32).reshape(cls_h.shape)
    want, _, want_idx = postproc.proposal_layer(prob, bbox_h, info, return_index=True)
    frac, ds, db = _match_rois(got, got_idx, want, want_idx)
    assert frac >= 0.995 and ds < 1e-6 and db < 1e-6, (frac, ds, db)
    want2, _, want2_idx = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info, return_index=True)
    assert want2.shape[0] == 1000
    frac, ds, db = _match_rois(got, got_idx, want2, want2_idx)
    print("bf16x3p e2e overlap %.4f  dscore %.2e  dbox %.2e" % (frac, ds, db))
    assert frac >= 0.999 and ds < 1e-5 and db < 2e-4, (frac, ds, db)
    assert rows_matched(got, want2) >= 0.999


def test_batch_of_four_equals_single_images(weights):
    """At 300x300 a batch of 4 runs the 1/16-scale layers row-stacked; each image's results must equal its own run."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x3p")
    ims = np.stack([synth.make_image(80 + i, 300, 300) for i in range(4)])
    cls_b, box_b = eng.forward_heads(torch.from_numpy(ims).cuda())
    batch = eng.detect_batch(ims)
    for i in range(4):
        c1, b1 = eng.forward_heads(torch.from_numpy(ims[i:i + 1]).cuda())
        assert torch.equal(c1[0], cls_b[i]) and torch.equal(b1[0], box_b[i])
        s, b = eng.detect(ims[i])
        np.testing.assert_array_equal(s, batch[i][0])
        np.testing.assert_array_equal(b, batch[i][1])


def test_reference_api_session_planes_5(weights):
    """get_network / Session(planes=5) / test_ctpn, the reference call sequence, on one image."""
    from ctpn_b200 import Session
    from lib.fast_rcnn.test import test_ctpn
    from lib.networks.factory import get_network
    sess = Session(weights, planes=5)
    net = get_network("VGGnet_test")
    im = synth.make_image(1, 600, 900)
    scores, boxes = test_ctpn(sess, net, im)
    blob, scale = net_cpu.image_blob(im)
    ref = net_cpu.forward(blob, weights)
    info = np.array([[blob.shape[1], blob.shape[2], scale]], np.float32)
    want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info)
    assert abs(scores.shape[0] - want.shape[0]) <= 2
    got = np.hstack([scores[:, None], boxes * np.float32(scale)])
    assert rows_matched(got, want) >= 0.995
