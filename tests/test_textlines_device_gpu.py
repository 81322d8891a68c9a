"""GPU: the batched device text-line connector (ctpn_text_lines / Engine.text_lines / Engine.detect_lines_images).  Every
comparison is np.array_equal on the float64 line arrays, with the same line counts, against the host connector
(ctpn_text_lines_host through textlines.text_lines) on the same inputs: boxes = float32(rois[:, 1:5] / float64 im_scale)."""
import numpy as np
import pytest
import torch

from ctpn_b200.textlines import text_lines
from oracle import synth

pytestmark = pytest.mark.gpu

SCALES = (1.0, 0.8333333333333334, 1.6, 600.0 / 1080)
RELAXED = (0.5, 0.3, 30, 0.6, 0.6, 0.3, 0.7, 8, 2)
# proposals past an image's count: they would fail the width check or form lines if the kernel read them
PAD_ROW = np.array([0.99, 5.0e4, 10.0, 5.0e4 + 16, 30.0], np.float32)


@pytest.fixture(scope="module")
def eng():
    from ctpn_b200 import Engine
    return Engine(None)


def to_rois(tp, sc, scale=1.0):
    """test_ctpn's inputs at blob scale: rois (score, boxes * scale) in float32"""
    tp = np.asarray(tp, np.float32).reshape(-1, 4)
    return np.concatenate([np.asarray(sc, np.float32).reshape(-1, 1), (tp * np.float32(scale)).astype(np.float32)], 1)


def host(r, hw, scale, mode, cfg=None):
    return text_lines(r[:, 1:5] / np.float64(scale), r[:, 0], hw, mode, cfg)


def run(eng, cases, mode, cfg=None, rows=None, out=None):
    """cases: [(rois [n,5], (h, w), im_scale)] -> host arrays (lines [B,rows,9], num [B], status [B])"""
    B = len(cases)
    rows = max(1, max(len(c[0]) for c in cases)) if rows is None else rows
    rois = np.tile(PAD_ROW, (B, rows, 1))
    cnt = np.zeros(B, np.int32)
    for b, (r, _, _) in enumerate(cases):
        rois[b, :len(r)] = r
        cnt[b] = len(r)
    lines, num, status = eng.text_lines(torch.from_numpy(rois).cuda(), torch.from_numpy(cnt).cuda(), [c[1] for c in cases],
                                        [c[2] for c in cases], mode, cfg, out=out)
    return lines.cpu().numpy(), num.cpu().numpy(), status.cpu().numpy()


def check(eng, cases, mode, cfg=None, rows=None, what=""):
    """device == host for every image of one batch; returns the number of lines"""
    lines, num, status = run(eng, cases, mode, cfg, rows)
    total = 0
    for b, (r, hw, s) in enumerate(cases):
        want = host(r, hw, s, mode, cfg)
        assert status[b] == 0, "%s image %d: status %d" % (what, b, status[b])
        assert num[b] == len(want), "%s image %d (%s): %d lines vs %d" % (what, b, mode, num[b], len(want))
        got = lines[b, :num[b]]
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), "%s image %d (%s)" % (what, b, mode)
        total += len(want)
    return total


@pytest.mark.parametrize("mode", ["H", "O"])
def test_golden_layouts(eng, mode):
    import os
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_postproc.npz"))
    cases = []
    for seed in range(4):
        tp, sc = synth.make_text_proposals(seed)
        cases.append((to_rois(tp, sc), (600, 900), 1.0))
    assert check(eng, cases, mode, what="golden") > 0
    lines, num, _ = run(eng, cases, mode)
    for seed in range(4):                         # and within float32 rounding of the reference's own output
        ref = gold["text_%s_%d" % (mode, seed)]
        assert num[seed] == len(ref) and np.abs(lines[seed, :num[seed]] - ref).max() <= 1e-4


@pytest.mark.parametrize("mode", ["H", "O"])
def test_random_layouts_sizes_and_scales(eng, mode):
    sizes = [(600, 900), (900, 600), (611, 1037)]
    cases = []
    for k in range(210):
        h, w = sizes[k % 3]
        tp, sc = synth.make_text_proposals(500 + k, im_h=h, im_w=w, n_lines=1 + k % 14, n_noise=20 + 5 * (k % 30))
        for s in SCALES:
            cases.append((to_rois(tp, sc, s), (h, w), s))
    total = 0
    for i in range(0, len(cases), 64):
        total += check(eng, cases[i:i + 64], mode, what="random batch %d" % (i // 64))
    print("%s: %d images, %d lines" % (mode, len(cases), total))
    assert total >= 300


def line_of(x0, n, y, h, step=16, width=16, score=0.95, drift=0.0, rs=None):
    """n proposals of a straight text line starting at x0"""
    out = []
    for k in range(n):
        yc = y + drift * k
        s = score if rs is None else float(rs.uniform(0.91, 0.99))
        out.append([s, x0 + step * k, yc - h / 2, x0 + step * k + width, yc + h / 2])
    return np.array(out, np.float32).reshape(-1, 5)


def edge_cases():
    rs = np.random.RandomState(7)
    tp, sc = synth.make_text_proposals(3)
    layout = to_rois(tp, sc)
    ties = layout.copy()
    ties[:, 0] = 0.99                                                   # saturated: every score equal
    rounded = layout.copy()
    rounded[:, 0] = np.round(rounded[:, 0], 1)
    merge = np.array([[0.95, 0, 100, 16, 130],                          # A: head, incompatible with B
                      [0.93, 10, 112, 26, 142],                         # B: head, one column nearer to S
                      [0.94, 32, 106, 48, 136],                         # S: successor of both -> shared tail
                      [0.94, 48, 106, 64, 136], [0.94, 64, 106, 80, 136], [0.92, 80, 106, 96, 136]], np.float32)
    gap = np.concatenate([line_of(0, 4, 300, 30, step=50),              # successors exactly max_gap = 50 apart
                          line_of(0, 4, 200, 30, step=51)])             # one column too far: no links
    same_x = np.array([[0.95, 100, 50 + 3 * k, 116, 80 + 3 * k] for k in range(5)], np.float32)
    two_box = np.concatenate([line_of(16 * k, 2, 40 + 45 * k, 20 + k, step=8 + 8 * (k % 3)) for k in range(10)])
    two_box[:, 2::2] += rs.uniform(-3, 3, (len(two_box), 2)).astype(np.float32)
    borders = np.concatenate([line_of(0, 5, 100, 24), line_of(900 - 1 - 64, 5, 200, 24)])
    borders[borders[:, 3] > 899, 3] = 899
    borders[-1, 1] = 899                                               # x1 = im_w - 1
    long_line = line_of(0, 160, 300, 28, drift=0.05, rs=rs)             # 160 members: the pairwise sum's recursive branch
    return [
        ("empty", np.zeros((0, 5), np.float32), (600, 900), 1.0),
        ("scores <= min_score", np.concatenate([layout[:, :1] * 0 + np.float32(0.7), layout[:, 1:]], 1), (600, 900), 1.0),
        ("low scores", np.concatenate([layout[:, :1] * 0.5, layout[:, 1:]], 1), (600, 900), 1.0),
        ("one proposal", layout[:1], (600, 900), 1.0),
        ("equal scores", ties, (600, 900), 1.0),
        ("rounded scores", rounded, (600, 900), 1.0),
        ("shuffled", layout[rs.permutation(len(layout))], (600, 900), 1.0),
        ("shuffled ties", ties[rs.permutation(len(ties))], (600, 900), 1.0),
        ("x1 = 0 and w - 1", borders, (600, 900), 1.0),
        ("gap = max_gap", gap, (600, 900), 1.0),
        ("merging chains", merge, (600, 900), 1.0),
        ("same x", same_x, (600, 900), 1.0),
        ("two-box chains", two_box, (600, 900), 1.0),
        ("160-member chain", long_line, (600, 2600), 1.0),
        ("160-member chain scaled", to_rois(long_line[:, 1:], long_line[:, 0], 1.6), (600, 2600), 1.6),
    ]


@pytest.mark.parametrize("mode", ["H", "O"])
def test_edge_cases(eng, mode):
    from ctpn_b200 import textlines
    cases = edge_cases()
    for name, r, hw, s in cases:
        check(eng, [(r, hw, s)], mode, what=name)
        check(eng, [(r, hw, s)], mode, cfg=RELAXED, what=name + " (relaxed cfg)")
    batch = [(r, hw, s) for _, r, hw, s in cases]
    check(eng, batch, mode, what="all edge cases in one batch")
    # the geometry does what the names say
    named = {name: (r, hw, s) for name, r, hw, s in cases}
    r = named["merging chains"][0]
    chains = textlines.groups(r[:, 1:5], r[:, 0], (600, 900))
    assert len(chains) == 2 and chains[0][1:] == chains[1][1:]
    gap = named["gap = max_gap"][0]
    assert len(textlines.groups(gap[:, 1:5], gap[:, 0], (600, 900))) == 1
    long_line = named["160-member chain"][0]
    assert max(len(c) for c in textlines.groups(long_line[:, 1:5], long_line[:, 0], (600, 2600))) > 128
    assert len(host(long_line, (600, 2600), 1.0, mode)) == 1


@pytest.mark.parametrize("mode", ["H", "O"])
def test_non_default_cfg_and_rows_above_1000(eng, mode):
    cases = []
    for k in range(8):
        tp, sc = synth.make_text_proposals(900 + k, n_lines=10, n_noise=40)
        cases.append((to_rois(tp, sc, SCALES[k % 4]), (600, 900), SCALES[k % 4]))
    for cfg in (RELAXED, (0.8, 0.1, 20, 0.8, 0.8, 1.0, 0.95, 16, 3), (0.0, 0.5, 80, 0.5, 0.5, 0.0, 0.0, 0, 0)):
        assert check(eng, cases, mode, cfg=cfg, what="cfg %s" % (cfg,)) >= 0
    big = []
    for k in range(3):
        tp, sc = synth.make_text_proposals(950 + k, im_w=2400, n_lines=40, n_noise=2500)
        assert len(sc) > 2500
        big.append((to_rois(tp, sc, 0.8), (600, 2400), 0.8))
    assert check(eng, big, mode, rows=4096, what="rows 4096") > 0
    assert check(eng, big, mode, cfg=RELAXED, rows=4096, what="rows 4096 relaxed") > 0


def test_batch_of_32_equals_images_alone_and_leaves_the_rest_unwritten(eng):
    from ctpn_b200 import Engine
    cases = []
    for k in range(32):
        tp, sc = synth.make_text_proposals(1200 + k, n_lines=1 + k % 9, n_noise=5 * k)
        cases.append((to_rois(tp, sc, SCALES[k % 4]), (600, 900), SCALES[k % 4]))
    rows = 1000
    packed = torch.full((32 * rows * 9 + 32,), float("nan"), dtype=torch.float64, device="cuda")
    lines_d, num_d, status_d = Engine.unpack_lines(packed, 32, rows)
    sentinel = lines_d.clone()
    run(eng, cases, "H", rows=rows, out=(lines_d, num_d, status_d))
    lines, num, status = lines_d.cpu().numpy(), num_d.cpu().numpy(), status_d.cpu().numpy()
    untouched = sentinel.cpu().numpy()
    assert len(set(num.tolist())) > 5 and (status == 0).all()
    for b, case in enumerate(cases):
        alone, n1, st1 = run(eng, [case], "H", rows=rows)
        assert st1[0] == 0 and n1[0] == num[b]
        assert np.array_equal(lines[b, :num[b]].view(np.uint64), alone[0, :num[b]].view(np.uint64)), b
        assert np.array_equal(lines[b, num[b]:].view(np.uint64), untouched[b, num[b]:].view(np.uint64)), b
    split = Engine.split_lines(lines_d, num_d, status_d)
    assert [len(x) for x in split] == num.tolist()


def test_proposal_outside_the_width_sets_status_and_raises(eng):
    from ctpn_b200 import CtpnError, Engine
    tp, sc = synth.make_text_proposals(2)
    good = to_rois(tp, sc)
    hot = good.copy()
    hot[:, 0] = 0.99
    cases = [(good, (600, 900), 1.0), (hot, (600, 100), 1.0), (good, (600, 900), 1.0)]
    with pytest.raises(RuntimeError, match="outside the image width"):
        host(hot, (600, 100), 1.0, "H")                               # the host connector raises on image 1
    lines, num, status = run(eng, cases, "H")
    assert status.tolist() == [0, 1, 0] and num[1] == 0
    want = host(good, (600, 900), 1.0, "H")
    for b in (0, 2):
        assert num[b] == len(want) and np.array_equal(lines[b, :num[b]], want)
    with pytest.raises(CtpnError, match="image 1: a proposal's x1 lies outside the image width 100"):
        Engine.split_lines(lines, num, status, im_hw=[c[1] for c in cases])
    # a count beyond the rows of the buffer: status 2 for that image only
    rois = torch.from_numpy(np.stack([good[:100], good[:100]])).cuda()
    lines, num, status = eng.text_lines(rois, torch.tensor([100, 101], dtype=torch.int32, device="cuda"), [(600, 900)] * 2,
                                        [1.0, 1.0])
    assert status.cpu().tolist() == [0, 2]
    with pytest.raises(CtpnError, match="image 1"):
        Engine.split_lines(lines, num, status)


# raw photo sizes: upscale to (600, 1000) u8; exact 1/2 u8; 16:9 and 3:1 -> float rescales of the blob; portrait; tiny
# upscale; f = 1
PHOTOS = [(240, 400), (1200, 1800), (360, 640), (300, 550), (200, 600), (450, 300), (37, 53), (600, 900)]
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 0, 0)      # synthetic weights score low: thresholds that let lines through


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.mark.parametrize("arith", ["f16f8", "bf16x2"])
def test_detect_lines_images_equals_rois_images_and_the_host_connector(weights, arith):
    from ctpn_b200 import Engine, frontend_plan
    e = Engine(weights, mode=arith)
    photos = [synth.make_image(600 + i, h, w) for i, (h, w) in enumerate(PHOTOS)]
    plan = frontend_plan(photos)
    assert {p.dtype for p in plan} == {"|u1", "<f4"}
    e.rois_images(photos, max_batch=32)                 # f16f8: the first batch calibrates the scales, then they are frozen
    lines_seen = 0
    for max_batch in (1, 7, 32):
        rois = e.rois_images(photos, max_batch=max_batch)
        for mode in ("H", "O"):
            for cfg in (None, LOW):
                got = e.detect_lines_images(photos, mode=mode, max_batch=max_batch, cfg=cfg)
                for i, p in enumerate(plan):
                    r, im_scale, f = rois[i]
                    want = text_lines(r[:, 1:5] / np.float64(im_scale), r[:, 0], p.resized, mode, cfg)
                    lines, f2 = got[i]
                    assert f2 == f == p.f
                    assert lines.shape == want.shape and np.array_equal(lines.view(np.uint64), want.view(np.uint64)), \
                        (arith, max_batch, mode, cfg, i)
                    lines_seen += len(want)
    assert lines_seen > 0
    with_images = e.detect_lines_images(photos, max_batch=3, return_resized=True, cfg=LOW)
    for (lines, f, resized), p, (l2, _) in zip(with_images, plan, e.detect_lines_images(photos, max_batch=3, cfg=LOW)):
        assert resized.shape[:2] == p.resized and np.array_equal(lines, l2)
    with pytest.raises(ValueError):
        e.detect_lines_images(photos, mode="X")
    with pytest.raises(ValueError):
        e.detect_lines_images(photos, max_batch=65)


def test_demo_device_lines_writes_the_native_connector_files(weights, tmp_path, monkeypatch):
    """ctpn/demo.py --batch 4 --device-frontend --device-lines == --batch 4 --device-frontend --native-connector: res_*.txt
    and the annotated images, byte for byte (connector thresholds lowered so that the synthetic weights give lines)."""
    import cv2
    from ctpn import demo
    from lib.text_connector.text_connect_cfg import Config
    for k, v in dict(TEXT_PROPOSALS_MIN_SCORE=0.05, MIN_V_OVERLAPS=0.5, MIN_SIZE_SIM=0.5, MIN_RATIO=0.0, LINE_MIN_SCORE=0.0,
                     TEXT_PROPOSALS_WIDTH=0, MIN_NUM_PROPOSALS=0).items():
        monkeypatch.setattr(Config, k, v)
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **weights)
    folder = tmp_path / "images"
    folder.mkdir()
    for i, (h, w) in enumerate([(300, 560), (1200, 1600), (480, 360), (200, 500), (240, 240), (350, 420)]):
        cv2.imwrite(str(folder / ("im_%d.png" % i)), synth.make_image(70 + i, h, w))
    out = {}
    for flag in ("--native-connector", "--device-lines"):
        res = tmp_path / ("results" + flag)
        monkeypatch.setattr(demo, "RESULTS_DIR", str(res))
        demo.main(["--weights", npz, "--planes", "2", "--images", str(folder / "*.png"), "--batch", "4", "--device-frontend", flag])
        out[flag] = {p.name: p.read_bytes() for p in sorted(res.iterdir())}
    a, b = out["--native-connector"], out["--device-lines"]
    assert len(a) == 12 and sorted(a) == sorted(b)
    assert any(v for k, v in a.items() if k.endswith(".txt")), "no text lines at all: the comparison would be vacuous"
    for name in a:
        assert a[name] == b[name], name
