"""GPU: the streamed device pipeline.  ctpn_resize_linear_u8_ragged_rows on row-compacted sources writes what
ctpn_resize_linear_u8_ragged writes on the whole images; Engine.stream_rois_images / stream_images / stream_lines_images
yield, in input order, what the list calls return, bit for bit, for any window and batch size; one streamed batch costs one
H2D and one result D2H, no synchronise of a stream or the device, and its upload overlaps the previous batch's kernels;
an early close leaves the engine usable; ctpn/demo.py --stream writes the files it writes without."""
import threading

import numpy as np
import pytest
import torch

from oracle import resize as R, synth

pytestmark = pytest.mark.gpu

# (h, w, f, row pitch - w): strong downscales of odd sizes, the camera-photo factor, exact 1/2 (INTER_AREA, also with odd
# sides: stored densely), just above 1/2, f = 1, an upscale
ROW_KERNEL_CASES = [(3024 // 2 + 1, 403, 0.198, 3), (1001, 333, 0.3, 0), (751, 1203, 0.4, 17), (1200, 900, 0.5, 0),
                    (301, 203, 0.5, 5), (1080, 611, 0.556, 1), (600, 450, 1.0, 0), (480, 641, 1.25, 9), (97, 55, 0.1, 2)]


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


def pack_rows(images, cases, compact, seed=0):
    """Sources back to back at row pitch w + pad, garbage in the pitch; compact: only frontend_rows of each image, and the
    row maps.  Returns (flat uint8, offsets, hwp, stored, maps int32, map offsets)."""
    from ctpn_b200.engine import frontend_rows
    rs = np.random.RandomState(seed)
    parts, offs, hwp, stored, maps, moffs, o, mo = [], [], [], [], [], [], 0, 0
    for im, (h, w, f, pad) in zip(images, cases):
        rows = frontend_rows(h, f, R.out_size(h, w, f, f)[0]) if compact else np.arange(h)
        block = rs.randint(0, 256, (len(rows), w + pad, 3)).astype(np.uint8)
        block[:, :w] = im[rows]
        m = rs.randint(-7, h + 7, h).astype(np.int32)          # rows that are not stored: anything
        m[rows] = np.arange(len(rows))
        parts.append(block.ravel())
        offs.append(o)
        hwp.append((h, w, w + pad))
        stored.append(len(rows))
        maps.append(m)
        moffs.append(mo)
        o += block.size
        mo += h
    return (np.concatenate(parts), np.array(offs, np.int64), np.array(hwp, np.int32), np.array(stored, np.int32),
            np.concatenate(maps), np.array(moffs, np.int64))


def run_rows_kernel(flat, offs, hwp, stored, maps, moffs, cases, sentinel=0xA5):
    from ctpn_b200 import _native as N
    fxy = np.array([[c[2], c[2]] for c in cases], np.float64)
    dst_hw = np.array([R.out_size(c[0], c[1], c[2], c[2]) for c in cases], np.int32)
    B, H, W = len(cases), int(dst_hw[:, 0].max()) + 3, int(dst_hw[:, 1].max()) + 5
    src, mp = torch.from_numpy(flat).cuda(), torch.from_numpy(maps).cuda()
    canvas = torch.full((B, H, W, 3), sentinel, dtype=torch.uint8, device="cuda")
    if stored is None:
        rc = N.lib.ctpn_resize_linear_u8_ragged(N.ptr(src), flat.size, N.ptr(offs), N.ptr(hwp), N.ptr(fxy), N.ptr(dst_hw), B, 3,
                                                N.ptr(canvas), H, W, N.stream_ptr())
    else:
        rc = N.lib.ctpn_resize_linear_u8_ragged_rows(N.ptr(src), flat.size, N.ptr(offs), N.ptr(hwp), N.ptr(stored), N.ptr(mp),
                                                     maps.size, N.ptr(moffs), N.ptr(fxy), N.ptr(dst_hw), B, 3, N.ptr(canvas), H, W,
                                                     N.stream_ptr())
    N.check(rc, "ragged resize")
    return canvas.cpu().numpy(), dst_hw


def test_compacted_sources_resize_like_the_whole_images():
    import cv2
    images = [synth.make_image(700 + i, h, w) for i, (h, w, _, _) in enumerate(ROW_KERNEL_CASES)]
    dense = pack_rows(images, ROW_KERNEL_CASES, compact=False)
    want, dst_hw = run_rows_kernel(dense[0], dense[1], dense[2], None, dense[4], dense[5], ROW_KERNEL_CASES)
    comp = pack_rows(images, ROW_KERNEL_CASES, compact=True)
    assert comp[3][0] < 0.42 * ROW_KERNEL_CASES[0][0] and comp[3][3] == 1200 and comp[3][4] == 301      # exact 1/2: every row
    for name, packed in (("compacted", comp), ("identity maps", dense)):
        got, _ = run_rows_kernel(*packed, ROW_KERNEL_CASES)
        for b, (dh, dw) in enumerate(dst_hw):
            what = "%s image %d %r" % (name, b, ROW_KERNEL_CASES[b])
            assert np.array_equal(got[b, :dh, :dw], want[b, :dh, :dw]), what
            assert (got[b, dh:] == 0xA5).all() and (got[b, :dh, dw:] == 0xA5).all(), what + ": padding was written"
    for b in (0, 2, 3, 7):
        f = ROW_KERNEL_CASES[b][2]
        assert np.array_equal(want[b, :dst_hw[b, 0], :dst_hw[b, 1]],
                              cv2.resize(images[b], None, None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR)), b


def test_a_map_entry_outside_the_stored_rows_is_clamped():
    """The map is device data: an entry below 0 or past the stored rows reads the first / last stored row instead."""
    cases = [(1001, 333, 0.3, 0), (97, 55, 0.1, 2)]
    images = [synth.make_image(720 + i, h, w) for i, (h, w, _, _) in enumerate(cases)]
    flat, offs, hwp, stored, maps, moffs = pack_rows(images, cases, compact=True)
    rs = np.random.RandomState(3)
    maps = maps.copy()
    hit = rs.rand(maps.size) < 0.3
    maps[hit] = rs.randint(-1000, 3000, int(hit.sum()))
    got, dst_hw = run_rows_kernel(flat, offs, hwp, stored, maps, moffs, cases)
    for b, (h, w, f, pad) in enumerate(cases):
        block = flat[offs[b]:offs[b] + stored[b] * (w + pad) * 3].reshape(stored[b], w + pad, 3)[:, :w]
        seen = block[np.clip(maps[moffs[b]:moffs[b] + h], 0, stored[b] - 1)]
        assert np.array_equal(got[b, :dst_hw[b, 0], :dst_hw[b, 1]], R.resize_linear_u8(seen, f)), b


# 40 photos: every branch of the front-end (upscale, exact 1/2, float rescale, portrait, tiny, f = 1) and, at 1700 x 2300
# and 2300 x 1700, sources that go up row-compacted
PHOTO_SIZES = [(240, 400), (1200, 1800), (300, 550), (200, 600), (450, 300), (37, 53), (600, 900), (1700, 2300), (2300, 1700),
               (1000, 3000)]


@pytest.fixture(scope="module")
def photos():
    return [synth.make_image(800 + i, *PHOTO_SIZES[i % len(PHOTO_SIZES)]) for i in range(40)]


def same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), i
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), i
            else:
                assert u == v, i


@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_streams_equal_the_list_calls(weights, photos, mode):
    from ctpn_b200 import Engine, frontend_plan
    eng = Engine(weights, mode=mode)
    assert sum(p.rows is not None for p in frontend_plan(photos)) == 8
    want = eng.rois_images(photos, return_resized=True)            # f16f8: the first batch calibrates the scales
    assert all(r[0].shape[0] > 0 for r in want)
    for window in (1, 7, 64):
        for max_batch in (1, 5, 32):
            got = list(eng.stream_rois_images((im for im in photos), max_batch=max_batch, return_resized=True, window=window))
            same(got, want)
    same(list(eng.stream_rois_images(iter(photos), window=7, max_batch=5)), [r[:3] for r in want])
    same(list(eng.stream_rois_images(iter(photos), window=7, max_batch=5, compact_rows=False)), [r[:3] for r in want])
    det = eng.detect_images(photos, return_resized=True)
    for window, max_batch in ((1, 1), (7, 5), (64, 32)):
        same(list(eng.stream_images((im for im in photos), max_batch=max_batch, return_resized=True, window=window)), det)
    for line_mode in ("H", "O"):
        lines = eng.detect_lines_images(photos, mode=line_mode, return_resized=True)
        assert sum(r[0].shape[0] for r in lines) > 0
        for window, max_batch in ((7, 5), (64, 32)):
            same(list(eng.stream_lines_images((im for im in photos), mode=line_mode, max_batch=max_batch, return_resized=True,
                                              window=window)), lines)
    assert not [t for t in threading.enumerate() if t.name.startswith("ctpn-stream-pack")]


def test_a_bad_image_raises_after_its_predecessors_and_the_engine_goes_on(weights, photos):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    want = eng.detect_images(photos[:12])
    mixed = photos[:9] + [photos[9].astype(np.float32)] + photos[10:12]
    got = []
    with pytest.raises(ValueError, match="image 9 must be HxWx3 uint8"):
        for r in eng.stream_images(iter(mixed), max_batch=4, window=6):
            got.append(r)
    same(got, want[:9])
    with pytest.raises(ValueError):
        eng.stream_images(photos, max_batch=65)
    with pytest.raises(ValueError):
        eng.stream_images(photos, window=0)
    # early close: the work in flight is waited for, the worker joined, and every other call still gives its results
    gen = eng.stream_images((im for im in photos), max_batch=4, window=8)
    same([next(gen) for _ in range(3)], eng.detect_images(photos[:3]))
    with pytest.raises(RuntimeError, match="still open"):
        next(eng.stream_images(iter(photos)))
    gen.close()
    assert not [t for t in threading.enumerate() if t.name.startswith("ctpn-stream-pack")]
    same(eng.detect_images(photos[:12]), want)
    same(list(eng.stream_images(iter(photos[:12]), max_batch=4, window=8)), want)


def test_a_streamed_batch_is_one_upload_one_download_and_no_synchronise(weights, photos):
    """torch.profiler census of a warm streamed run: per batch one H2D and one D2H, the host waits on events only, and
    uploads run while the previous batch's kernels do.  The number of batches comes from the plan, not from the trace,
    and a short streamed run goes first inside the profile: the profiler can lose the first device records after it
    starts (seen here: the first upload and resize kernel of a run, when other profiles had run in the process)."""
    from torch.profiler import ProfilerActivity, profile, record_function
    from ctpn_b200 import Engine, frontend_plan, ragged_plan
    eng = Engine(weights, mode="f16f8")
    batches = 0
    for k in range(0, len(photos), 12):
        plan = frontend_plan(photos[k:k + 12])
        batches += len(ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 4))
    assert batches >= 10

    def run(ims=photos):
        return list(eng.stream_rois_images(iter(ims), max_batch=4, window=12))

    want = run()                        # warm: calibration, workspaces, slot buffers
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(photos[:4])
        torch.cuda.synchronize()
        with record_function("streamed_run"):
            got = run()
    same(got, want)
    span = next(e for e in prof.events() if e.name == "streamed_run").time_range
    inside = [e for e in prof.events() if span.start <= e.time_range.start <= span.end]
    during = [e.name for e in inside]

    def starts(events):
        return [round((e.time_range.start - span.start) / 1e3, 2) for e in events]

    dev = [e for e in inside if "cuda" in str(e.device_type).lower()]
    uploads = [e for e in dev if e.name.startswith("Memcpy HtoD")]
    downloads = [e for e in dev if e.name.startswith("Memcpy DtoH")]
    resizes = [e for e in dev if "resize_linear_u8_ragged" in e.name and "kernel" in e.name]
    what = "%d batches; ms from the run's start: H2D %s, D2H %s, resize kernels %s" % (batches, starts(uploads), starts(downloads),
                                                                                      starts(resizes))
    assert len(uploads) == len(downloads) == len(resizes) == batches, what
    assert during.count("cudaStreamSynchronize") <= 3         # the end of the stream: its three streams, once each
    assert during.count("cudaDeviceSynchronize") == 0
    assert during.count("cudaEventSynchronize") >= batches
    kernels = [e for e in dev if not e.name.startswith(("Memcpy", "Memset"))]
    overlapped = sum(1 for c in uploads if any(k.time_range.start < c.time_range.end and c.time_range.start < k.time_range.end
                                               for k in kernels))
    assert overlapped >= batches // 2, (overlapped, what)


def test_demo_stream_writes_the_same_files(weights, tmp_path, monkeypatch):
    """ctpn/demo.py --batch 4 --device-frontend [--device-lines] --stream == the same without --stream, byte for byte."""
    import cv2
    from ctpn import demo
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **weights)
    folder = tmp_path / "images"
    folder.mkdir()
    prev = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        for i, (h, w) in enumerate([(300, 560), (1200, 1600), (480, 360), (200, 500), (1700, 2300), (350, 420)]):
            cv2.imwrite(str(folder / ("im_%d.png" % i)), synth.make_image(70 + i, h, w))
        for lines in ([], ["--device-lines"]):
            out = {}
            for stream in ([], ["--stream"]):
                res = tmp_path / ("results_%d_%d" % (len(lines), len(stream)))
                monkeypatch.setattr(demo, "RESULTS_DIR", str(res))
                demo.main(["--weights", npz, "--planes", "2", "--images", str(folder / "*.png"), "--batch", "4",
                           "--device-frontend"] + lines + stream)
                out[len(stream)] = {p.name: p.read_bytes() for p in sorted(res.iterdir())}
            assert len(out[0]) == 12 and sorted(out[0]) == sorted(out[1])
            for name in out[0]:
                assert out[0][name] == out[1][name], (lines, name)
    finally:
        cv2.ipp.setUseIPP(prev)
    with pytest.raises(SystemExit):
        demo.main(["--batch", "4", "--stream"])
