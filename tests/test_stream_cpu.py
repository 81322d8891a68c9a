"""CPU: the host side of the streamed device pipeline (Engine.stream_rois_images).  frontend_rows lists exactly the source
rows the oracle's restatement of cv2.resize reads; the upload layout and packing keep every such row reachable through
the row map; ctpn_resize_linear_u8_ragged_rows rejects every bad descriptor before any CUDA call; and the window /
ordering / shutdown logic of the pipeline driver holds on stages that need no device."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from ctpn_b200 import _native as N
from ctpn_b200.engine import (StreamBatch, frontend_plan, frontend_rows, run_stream, stream_layout, stream_pack,
                              stream_windows)
from oracle import resize as R


# ---- frontend_rows ----------------------------------------------------------------------------------------------------

def brute_force_rows(h, f, out_h):
    """Every row index the oracle's row taps name, one output row at a time."""
    s0, s1, _, _ = R._taps(out_h, h, 1.0 / f, False)
    return sorted(set(int(v) for v in s0) | set(int(v) for v in s1))


ROW_CASES = [(3024, 600 / 3024.0), (4032, 1200 / 4032.0), (1080, 600 / 1080.0), (1000, 0.4), (600, 1.0), (240, 2.5), (37, 600 / 37.0),
             (301, 0.3), (1, 3.0), (2, 0.7), (2, 4.0), (1, 1.0), (999, 0.1), (1001, 1 / 3.0), (768, 600 / 768.0), (50, 0.02)]


@pytest.mark.parametrize("h,f", ROW_CASES)
def test_rows_equal_a_brute_force_enumeration(h, f):
    out_h = R.out_size(h, h, f, f)[0]
    rows = frontend_rows(h, f, out_h)
    assert rows.dtype == np.int64 and list(rows) == brute_force_rows(h, f, out_h)
    assert rows[0] >= 0 and rows[-1] <= h - 1 and (np.diff(rows) > 0).all()


def test_rows_clamp_at_the_last_row_and_cover_an_upscale():
    assert list(frontend_rows(10, 0.3, 3)) == brute_force_rows(10, 0.3, 3)
    assert list(frontend_rows(4, 1.0, 4)) == [0, 1, 2, 3]                 # row 3's second tap is clamped onto row 3
    assert list(frontend_rows(37, 4.0, 148)) == list(range(37))          # an upscale reads every row
    assert list(frontend_rows(600, 1.0, 600)) == list(range(600))
    assert list(frontend_rows(1, 2.0, 2)) == [0] and list(frontend_rows(2, 1.5, 3)) == [0, 1]


def test_exact_half_is_dense():
    assert list(frontend_rows(1200, 0.5, 600)) == list(range(1200))
    assert list(frontend_rows(301, 0.5, 150)) == list(range(301))
    assert frontend_plan([(1200, 1800)])[0].rows is None


def test_live_fraction_of_a_camera_photo():
    p = frontend_plan([(3024, 4032)])[0]
    assert p.rows == tuple(frontend_rows(3024, p.f, p.resized[0]))
    assert 0.39 <= len(p.rows) / 3024.0 <= 0.41
    q = frontend_plan([(4032, 3024)])[0]
    assert 0.39 <= len(q.rows) / 4032.0 <= 0.41


def test_compaction_needs_a_quarter_of_the_rows_gone():
    for shape, compacted in [((3024, 4032), True), ((1000, 3000), False), ((1080, 1920), False), ((768, 1024), False),
                             ((480, 640), False), ((600, 900), False), ((2000, 3000), True), ((1500, 2000), False)]:
        p = frontend_plan([shape])[0]
        assert (p.rows is not None) == compacted, shape
        if compacted:
            assert 4 * len(p.rows) <= 3 * shape[0]
    # 1500 -> 600 keeps 1199 of 1500 rows: under a quarter gone, so the image goes up whole
    assert len(frontend_rows(1500, 0.4, 600)) > 0.75 * 1500


def test_plan_numbers_images_from_first():
    with pytest.raises(ValueError, match="image 7 "):
        frontend_plan([(600, 900), (1, 5000, 3)], first=6)


# ---- layout and packing -----------------------------------------------------------------------------------------------

def _batch(shapes, seed=0):
    rs = np.random.RandomState(seed)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    items = frontend_plan(images)
    return StreamBatch(list(range(len(images))), items, images, (max(p.blob[0] for p in items), max(p.blob[1] for p in items)))


def test_packed_rows_give_the_resize_of_the_whole_image():
    batch = _batch([(1813, 2417), (300, 450), (2400, 1700)])          # compacted, dense (upscale), compacted
    assert [p.rows is not None for p in batch.items] == [True, False, True]
    lay = stream_layout(batch.items, [im.shape[:2] for im in batch.images])
    assert lay.map_base % 4 == 0 and lay.sizes_at == lay.map_base + 4 * (1813 + 300 + 2400) and lay.total == lay.sizes_at + 28 * 3
    buf = np.full(lay.total + 5, 0xA5, np.uint8)
    stream_pack(buf, lay, batch)
    assert (buf[lay.total:] == 0xA5).all()
    for k, (im, p) in enumerate(zip(batch.images, batch.items)):
        h, w = im.shape[:2]
        n = int(lay.stored[k])
        stored = buf[lay.offsets[k]:lay.offsets[k] + n * w * 3].reshape(n, w, 3)
        m = buf[lay.map_base + 4 * lay.maps[k]:lay.map_base + 4 * (lay.maps[k] + h)].view(np.int32)
        assert n == (h if p.rows is None else len(p.rows)) and 0 <= m.min() and m.max() < n
        seen = stored[m]                      # what the kernel sees of each original row
        live = frontend_rows(h, p.f, p.resized[0])
        assert np.array_equal(seen[live], im[live])
        assert np.array_equal(R.resize_linear_u8(seen, p.f), R.resize_linear_u8(im, p.f))
    B = 3
    tail = buf[lay.sizes_at:lay.total]
    blobs = np.array([p.blob for p in batch.items], np.int32)
    assert np.array_equal(tail[:8 * B].view(np.int32).reshape(B, 2), blobs)
    assert np.array_equal(tail[8 * B:16 * B].view(np.int32).reshape(B, 2), blobs >> 4)
    info = tail[16 * B:].view(np.float32).reshape(B, 3)
    assert np.array_equal(info, np.array([[p.blob[0], p.blob[1], p.im_scale] for p in batch.items], np.float32))


def test_a_batch_without_compacted_images_has_no_maps():
    batch = _batch([(480, 640), (768, 1024)])
    lay = stream_layout(batch.items, [im.shape[:2] for im in batch.images])
    assert lay.maps is None and lay.sizes_at == lay.map_base and list(lay.stored) == [480, 768]
    batch = _batch([(1813, 2417), (2400, 1700)])
    dense = stream_layout(batch.items, [im.shape[:2] for im in batch.images], compact_rows=False)
    assert dense.maps is None and list(dense.stored) == [1813, 2400] and dense.rows == [None, None]
    assert stream_layout(batch.items, [im.shape[:2] for im in batch.images]).total < 0.72 * dense.total


# ---- ctpn_resize_linear_u8_ragged_rows: validation before any CUDA call --------------------------------------------

FAKE = C.c_void_p(0x1000)        # a non-null "device" pointer: validation fails before anything dereferences it


def descriptors():
    """Three images packed back to back: 100 x 60 holding 41 of its rows, 30 x 50 whole at pitch 56, 64 x 96 whole."""
    srcs = [(100, 60, 60, 0.2, 41), (30, 50, 56, 0.5, 30), (64, 96, 96, 1.0, 64)]
    offs, o = [], 0
    for h, w, pitch, f, stored in srcs:
        offs.append(o)
        o += stored * pitch * 3
    return dict(elems=o, offs=np.array(offs, np.int64), hwp=np.array([s[:3] for s in srcs], np.int32),
                stored=np.array([s[4] for s in srcs], np.int32), map_elems=100 + 30 + 64, maps=np.array([0, 100, 130], np.int64),
                fxy=np.array([[s[3], s[3]] for s in srcs], np.float64),
                dst=np.array([R.out_size(s[0], s[1], s[3], s[3]) for s in srcs], np.int32), B=3, H=64, W=96)


def call(d, src=FAKE, dst=FAKE, row_map=FAKE, null=()):
    a = {k: (None if k in null else N.ptr(d[k])) for k in ("offs", "hwp", "stored", "maps", "fxy", "dst")}
    rc = N.lib.ctpn_resize_linear_u8_ragged_rows(src, d["elems"], a["offs"], a["hwp"], a["stored"], row_map, d["map_elems"],
                                                 a["maps"], a["fxy"], a["dst"], d["B"], d.get("C", 3), dst, d["H"], d["W"], None)
    return rc, N.last_error()


def test_valid_descriptors_stop_at_the_device_query():
    import torch
    if torch.cuda.is_available():
        pytest.skip("the call would launch on the fake pointers; only meaningful without a GPU")
    rc, msg = call(descriptors())
    assert rc == N.ERR_NO_DEVICE, msg


def test_null_pointers_are_invalid():
    d = descriptors()
    for kw in (dict(src=None), dict(dst=None), dict(row_map=None)):
        rc, msg = call(d, **kw)
        assert rc == N.ERR_INVALID and "null" in msg, kw
    for name in ("offs", "hwp", "stored", "maps", "fxy", "dst"):
        rc, msg = call(d, null=(name,))
        assert rc == N.ERR_INVALID and "null" in msg, name


@pytest.mark.parametrize("bad", [0, -1, 101])
def test_stored_rows_within_the_source_height(bad):
    d = descriptors()
    d["stored"][0] = bad
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "stored rows" in msg


def test_the_stored_extent_must_lie_within_src_elems():
    d = descriptors()
    d["elems"] -= 1                        # image 2 ends exactly at the end of the packed sources
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "src_elems" in msg
    d = descriptors()
    d["stored"][2] = 64
    d["stored"][0] = 42                    # one more row than was packed: image 0 itself still fits, the last image no longer...
    d["offs"][1:] += 60 * 3
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "src_elems" in msg
    d = descriptors()
    d["offs"][1] = -3
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1" in msg
    d = descriptors()
    d["offs"][0] = 1 << 62                 # no wrap-around in the extent arithmetic
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg


def test_the_row_map_must_lie_within_map_elems():
    d = descriptors()
    d["map_elems"] -= 1                    # a map has one entry per ORIGINAL row: image 2's 64 entries end at 194
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "row map" in msg
    for b, off in ((1, -1), (0, 1 << 62), (1, 165)):
        d = descriptors()
        d["maps"][b] = off
        rc, msg = call(d)
        assert rc == N.ERR_INVALID and "image %d" % b in msg and "row map" in msg, (b, off)


def test_pitch_size_scale_batch_and_channels_as_in_the_dense_call():
    d = descriptors()
    d["hwp"][1, 2] = 49
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1" in msg and "pitch" in msg
    d = descriptors()
    d["dst"][0, 0] += 1                    # the output size follows the ORIGINAL height, not the stored one
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "cv2 would produce" in msg
    d = descriptors()
    d["W"] = 95
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "canvas" in msg
    for bad in (0.0, -0.5, float("nan")):
        d = descriptors()
        d["fxy"][1, 1] = bad
        rc, msg = call(d)
        assert rc == N.ERR_INVALID and "image 1" in msg
    for B in (0, 65):
        d = descriptors()
        d["B"] = B
        rc, msg = call(d)
        assert rc == N.ERR_INVALID and "B = %d" % B in msg
    for ch in (0, 5):
        d = descriptors()
        d["C"] = ch
        rc, msg = call(d)
        assert rc == N.ERR_INVALID and "channel" in msg


# ---- the pipeline driver on stages without a device ----------------------------------------------------------------------

class StubStages:
    """run_stream's stages on the host: the 'result' of an image is (its stream index, its first pixel).  Records what
    ran where, and checks the slot discipline: a slot is packed only after its previous upload, uploaded only after its
    previous compute."""

    def __init__(self, pack_delay=0.0):
        self.calls, self.pack_threads, self.drained, self.pack_delay = [], set(), 0, pack_delay
        self.state = {0: "free", 1: "free"}
        self.main = threading.get_ident()

    def stage(self, batch, slot):
        assert threading.get_ident() == self.main
        return ("staged", tuple(batch.idxs))

    def pack(self, batch, slot, staged):
        assert staged == ("staged", tuple(batch.idxs))
        self.pack_threads.add(threading.current_thread().name)
        time.sleep(self.pack_delay)
        return [int(im[0, 0, 0]) for im in batch.images]

    def upload(self, batch, slot, packed):
        assert threading.get_ident() == self.main
        self.calls.append(("upload", tuple(batch.idxs), slot))
        return packed

    def compute(self, batch, slot, uploaded):
        self.calls.append(("compute", tuple(batch.idxs), slot))
        return uploaded

    def finish(self, batch, handle):
        self.calls.append(("finish", tuple(batch.idxs)))
        return [(i, v) for i, v in zip(batch.idxs, handle)]

    def drain(self):
        self.drained += 1

    def run(self, images, window, max_batch):
        def prepare(im, index):
            return im, frontend_plan([im], first=index)[0]
        return run_stream(stream_windows(images, window, max_batch, prepare), self.stage, self.pack, self.upload, self.compute,
                          self.finish, self.drain)


SHAPES = [(48, 64), (64, 48), (30, 90), (60, 60), (100, 40), (33, 47)]


def photos(n, bad_at=None):
    """A generator (not a list) of n small images whose first pixel is their index; image bad_at is float32."""
    for i in range(n):
        h, w = SHAPES[i % len(SHAPES)]
        im = np.zeros((h, w, 3), np.float32 if i == bad_at else np.uint8)
        im[0, 0, 0] = i % 251
        yield im


def packer_threads():
    return [t for t in threading.enumerate() if t.name.startswith("ctpn-stream-pack")]


@pytest.mark.parametrize("window", [1, 2, 7, 64])
@pytest.mark.parametrize("max_batch", [1, 3, 32])
@pytest.mark.parametrize("n", [0, 1, 5, 23])
def test_results_come_in_input_order_for_any_window(window, max_batch, n):
    st = StubStages()
    got = list(st.run(photos(n), window, max_batch))
    assert got == [(i, i % 251) for i in range(n)]
    assert st.drained == 1 and not packer_threads()
    computed = [c[1] for c in st.calls if c[0] == "compute"]
    assert sorted(i for b in computed for i in b) == list(range(n)) and all(len(b) <= min(window, max_batch) for b in computed)
    assert all(max(b) // window == min(b) // window for b in computed)          # a batch never spans two windows
    assert st.pack_threads <= {"ctpn-stream-pack_0"}
    # slots alternate, every batch is uploaded before it is computed and computed before it is finished, and batch k + 1
    # is uploaded before batch k is finished
    order = {(c[0], c[1]): j for j, c in enumerate(st.calls)}
    for k, b in enumerate(computed):
        assert ("compute", b, k & 1) in st.calls and order[("upload", b)] < order[("compute", b)] < order[("finish", b)]
        if k + 1 < len(computed):
            assert order[("upload", computed[k + 1])] < order[("finish", b)]


def test_any_iterable_is_taken():
    ims = list(photos(9))
    for source in (ims, tuple(ims), iter(ims), (im for im in ims)):
        assert [r[0] for r in StubStages().run(source, 4, 2)] == list(range(9))


def test_an_iterable_is_pulled_a_window_at_a_time():
    pulled = []

    def source():
        for i, im in enumerate(photos(40)):
            pulled.append(i)
            yield im

    gen = StubStages().run(source(), 4, 2)
    assert next(gen) == (0, 0)
    assert len(pulled) <= 3 * 4           # the window being yielded and the two batches packed and uploaded ahead of it
    gen.close()
    assert len(pulled) <= 3 * 4 and not packer_threads()


@pytest.mark.parametrize("window,max_batch", [(1, 1), (4, 2), (64, 32), (5, 32)])
@pytest.mark.parametrize("bad_at", [0, 3, 10, 16])
def test_a_bad_image_raises_after_its_predecessors(window, max_batch, bad_at):
    st = StubStages()
    gen = st.run(photos(17, bad_at=bad_at), window, max_batch)
    got = []
    with pytest.raises(ValueError, match="image %d must be HxWx3 uint8" % bad_at):
        for r in gen:
            got.append(r[0])
    assert got == list(range(bad_at))
    assert st.drained == 1 and not packer_threads()
    assert list(gen) == []


def test_close_joins_the_worker_and_drains():
    st = StubStages(pack_delay=0.02)
    gen = st.run(photos(30), 6, 3)
    assert [next(gen)[0] for _ in range(4)] == [0, 1, 2, 3]
    assert packer_threads()
    gen.close()
    assert st.drained == 1 and not packer_threads()
    unstarted = StubStages()
    unstarted.run(photos(5), 2, 2).close()          # never started: nothing to join, nothing to drain
    assert unstarted.drained == 0 and not packer_threads()


def test_a_failing_stage_still_joins_and_drains():
    st = StubStages()

    def compute(batch, slot, uploaded):
        if 7 in batch.idxs:
            raise RuntimeError("boom")
        return uploaded

    st.compute = compute
    with pytest.raises(RuntimeError, match="boom"):
        list(st.run(photos(12), 4, 2))
    assert st.drained == 1 and not packer_threads()
