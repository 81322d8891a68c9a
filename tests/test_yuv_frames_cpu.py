"""CPU: the host side of YUV 4:2:0 video frames in device memory.  oracle/yuv.py equals cv2.cvtColor on every (Y, U, V)
triple and on frames in all four layouts; ctpn_resize_linear_u8_yuv420 rejects every bad descriptor before any CUDA call;
the YUV420 constructors give descriptors that read the frame's planes for every layout a caller will have; and the rules
of the raw-photo calls -- one kind of image per call, planes on the engine's device, even sides, BGR only -- hold without
a device."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from ctpn_b200 import YUV420
from ctpn_b200 import _native as N
from ctpn_b200.engine import (FRAME, HOST, TENSOR, StreamBatch, frontend_plan, images_on_device, on_device, stream_layout,
                              stream_pack, yuv420_descriptor)
from oracle import resize as R, yuv

FAKE = 0x10000        # a non-null "device" address: validation fails before anything dereferences it
CODES = {"NV12": cv2.COLOR_YUV2BGR_NV12, "NV21": cv2.COLOR_YUV2BGR_NV21, "I420": cv2.COLOR_YUV2BGR_I420,
         "YV12": cv2.COLOR_YUV2BGR_YV12}


# ---- the oracle against cv2.cvtColor -------------------------------------------------------------------------------------

def test_oracle_equals_cvtcolor_on_every_yuv_triple():
    """All 2^24 (Y, U, V): a 512 x 512 frame whose 256 x 256 chroma planes hold every (U, V) pair and whose 2 x 2 luma
    blocks hold 4 luma values, 64 frames for the 256 luma values; through the NV12 and the I420 code."""
    U = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 256, 1)
    V = np.ascontiguousarray(U.T)
    bad = 0
    for k in range(64):
        Y = np.tile((4 * k + np.arange(4, dtype=np.uint8)).reshape(2, 2), (256, 256))
        want = yuv.yuv_to_bgr(Y, U, V)
        for layout in ("NV12", "I420"):
            bad += int((cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, layout), CODES[layout]) != want).sum())
    assert bad == 0


@pytest.mark.parametrize("h,w", [(2, 2), (4, 6), (34, 1002), (102, 66), (480, 640)])
def test_oracle_equals_cvtcolor_in_every_layout(h, w):
    rng = np.random.default_rng(h * 7 + w)
    Y = rng.integers(0, 256, (h, w), dtype=np.uint8)
    U = rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8)
    V = rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8)
    want = yuv.yuv_to_bgr(Y, U, V)
    for layout in yuv.LAYOUTS:
        buf = yuv.planes_to_buffer(Y, U, V, layout)
        assert np.array_equal(cv2.cvtColor(buf, CODES[layout]), want), layout
        assert all(np.array_equal(a, b) for a, b in zip(yuv.buffer_to_planes(buf, layout), (Y, U, V))), layout
    assert np.array_equal(cv2.cvtColorTwoPlane(Y, np.stack([U, V], -1), cv2.COLOR_YUV2BGR_NV12), want)


# ---- ctpn_resize_linear_u8_yuv420: validation before any CUDA call --------------------------------------------------------

def descriptors():
    """Three frames, planes (Y, U, V) each with the stated allocation size its box ends at:
      0  a dense 100 x 60 NV12 buffer (U and V interleaved after the luma),
      1  a 30 x 50 frame in three allocations: luma at pitch 64, U at pitch 32, V read bottom-up, right to left,
      2  a 64 x 96 NV21 crop at row 2, column 4 of a 128-byte-pitch surface with chroma in an allocation of its own."""
    planes = np.array([FAKE] * 3 + [FAKE + (1 << 24), FAKE + (2 << 24), FAKE + (3 << 24)] +
                      [FAKE + (4 << 24), FAKE + (5 << 24), FAKE + (5 << 24)], np.uint64)
    nbytes = np.array([6000, 6000 + 49 * 60 + 29 * 2 + 1, 9000,
                       29 * 64 + 50, 14 * 32 + 25, 14 * 32 + 25,
                       260 + 63 * 128 + 96, 1 + 31 * 128 + 47 * 2 + 1, 31 * 128 + 47 * 2 + 1], np.uint64)
    offs = np.array([0, 6000, 6001, 0, 0, 14 * 32 + 24, 2 * 128 + 4, 1, 0], np.int64)
    strides = np.array([[60, 1], [60, 2], [60, 2], [64, 1], [32, 1], [-32, -1], [128, 1], [128, 2], [128, 2]], np.int64)
    return dict(planes=planes, nbytes=nbytes, offs=offs, strides=strides,
                hw=np.array([[100, 60], [30, 50], [64, 96]], np.int32),
                fxy=np.array([[0.2, 0.2], [0.5, 0.5], [1.0, 1.0]], np.float64),
                dst=np.array([R.out_size(100, 60, 0.2, 0.2), R.out_size(30, 50, 0.5, 0.5), R.out_size(64, 96, 1.0, 1.0)],
                             np.int32),
                B=3, H=64, W=96)


ARRAYS = ("planes", "nbytes", "offs", "strides", "hw", "fxy", "dst")


def call(d, dst=C.c_void_p(FAKE), null=()):
    a = {k: (None if k in null else N.ptr(np.ascontiguousarray(d[k]))) for k in ARRAYS}
    rc = N.lib.ctpn_resize_linear_u8_yuv420(a["planes"], a["nbytes"], a["offs"], a["strides"], a["hw"], a["fxy"], a["dst"],
                                            d["B"], dst, d["H"], d["W"], None)
    return rc, N.last_error()


def tile(d, B):
    """The three frames of d repeated to B frames."""
    d = dict(d)
    reps = -(-B // 3)
    for k, per in (("planes", 3), ("nbytes", 3), ("offs", 3), ("strides", 3), ("hw", 1), ("fxy", 1), ("dst", 1)):
        d[k] = np.concatenate([d[k]] * reps)[:B * per]
    d["B"] = B
    return d


@pytest.mark.parametrize("B", [3, 32, 33, 64])
def test_valid_descriptors_stop_at_the_device_query(B):
    if torch.cuda.is_available():
        pytest.skip("the call would launch on the fake pointers; only meaningful without a GPU")
    rc, msg = call(tile(descriptors(), B))
    assert rc == N.ERR_NO_DEVICE, msg


@pytest.mark.parametrize("B", [0, -1, 65])
def test_batch_size_within_1_to_64(B):
    d = tile(descriptors(), 65)
    d["B"] = B
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "B = %d" % B in msg


def test_null_pointers_are_invalid():
    d = descriptors()
    rc, msg = call(d, dst=None)
    assert rc == N.ERR_INVALID and "null" in msg
    for name in ARRAYS:
        rc, msg = call(d, null=(name,))
        assert rc == N.ERR_INVALID and "null" in msg, name
    for i in range(9):
        d = descriptors()
        d["planes"][i] = 0
        rc, msg = call(d)
        assert rc == N.ERR_INVALID and "image %d: null %s plane" % (i // 3, "YUV"[i % 3]) in msg, msg


@pytest.mark.parametrize("hw", [(101, 60), (100, 61), (1, 60), (0, 60), (100, -2)])
def test_sides_must_be_even_and_positive(hw):
    d = descriptors()
    d["hw"][0] = hw
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "even and positive" in msg


@pytest.mark.parametrize("i", range(9))
def test_each_plane_must_end_inside_its_allocation(i):
    d = descriptors()
    d["nbytes"][i] -= 1                    # each plane's highest byte is the last byte of its allocation
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image %d: the %s plane" % (i // 3, "YUV"[i % 3]) in msg and "outside" in msg, msg


@pytest.mark.parametrize("i", range(9))
def test_each_plane_must_start_inside_its_allocation(i):
    d = descriptors()
    h, w = d["hw"][i // 3] // (2 if i % 3 else 1)
    lowest = d["offs"][i] + sum(min(0, int(n - 1) * int(s)) for n, s in zip((h, w), d["strides"][i]))
    assert lowest >= 0                     # frame 1's V plane reaches byte 0 through its negative strides
    d["offs"][i] -= lowest + 1             # the highest byte moves down with it: only the lowest leaves the allocation
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image %d: the %s plane" % (i // 3, "YUV"[i % 3]) in msg and "outside" in msg, msg


def test_zero_strides_broadcast():
    d = descriptors()
    d["strides"][4] = [0, 0]               # frame 1's U plane: one byte, read everywhere
    d["offs"][4], d["nbytes"][4] = 0, 1
    rc, msg = call(d)
    assert "image 1" not in msg, msg
    d["offs"][4] = 1
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1: the U plane" in msg


@pytest.mark.parametrize("stride", [1 << 62, -(1 << 62), (1 << 63) - 1])
def test_the_extent_arithmetic_does_not_wrap(stride):
    d = descriptors()
    d["strides"][0][0] = stride            # 99 rows of it: far outside any int64
    d["nbytes"][0] = (1 << 64) - 1
    d["offs"][0] = (1 << 63) - 1 if stride < 0 else 0
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0: the Y plane" in msg and "outside" in msg
    d = descriptors()
    d["offs"][8] = (1 << 63) - 1           # offset alone at the end of the int64 range
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2: the V plane" in msg


@pytest.mark.parametrize("i", [0, 4, 8])
def test_column_strides_fit_32_bits(i):
    d = descriptors()
    d["strides"][i][1] = 1 << 31
    d["nbytes"][i] = 1 << 40
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image %d: %s plane column stride" % (i // 3, "YUV"[i % 3]) in msg and "32-bit" in msg


def test_sizes_scales_dst_and_canvas():
    d = descriptors()
    d["fxy"][2] = [0.0, 1.0]
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "scale" in msg
    d = descriptors()
    d["fxy"][1] = [1e9, 1e9]
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1" in msg and "too large" in msg
    d = descriptors()
    d["dst"][0] = [d["dst"][0][0] + 1, d["dst"][0][1]]       # not what cv2 would produce
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "cv2 would produce" in msg
    d = descriptors()
    d["W"] = 95                            # frame 2's 96 columns do not fit
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "canvas" in msg
    d = descriptors()
    d["H"] = 0
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "canvas" in msg


# ---- the constructors' descriptors ---------------------------------------------------------------------------------------

def storage_bytes(t):
    st = t.untyped_storage()
    return torch.empty(0, dtype=torch.uint8).set_(st, 0, (st.nbytes(),), (1,)).numpy().copy()


def read_back(frame):
    """The Y, U, V planes the kernel reads through the frame's descriptor: sample (y, x) of plane p at byte
    offset + y * row_stride + x * col_stride of its allocation (a host copy of the storage bytes)."""
    H, W = frame.shape[:2]
    out = []
    for (addr, nbytes, off, (rs, cs)), p, (h, w) in zip(yuv420_descriptor(frame), frame, [(H, W)] + [(H // 2, W // 2)] * 2):
        st = p.untyped_storage()
        assert addr == st.data_ptr() and nbytes == st.nbytes()
        y, x = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        idx = off + y * rs + x * cs
        assert idx.min() >= 0 and idx.max() < nbytes
        out.append(storage_bytes(p)[idx])
    return out


def random_planes(rng, h, w):
    return (rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8),
            rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8))


def frames():
    """(name, frame, the BGR image cv2.cvtColor gives for it)."""
    rng = np.random.default_rng(11)
    h, w = 34, 58
    Y, U, V = random_planes(rng, h, w)
    bgr = yuv.yuv_to_bgr(Y, U, V)
    for layout in yuv.LAYOUTS:
        buf = yuv.planes_to_buffer(Y, U, V, layout)
        assert np.array_equal(cv2.cvtColor(buf, CODES[layout]), bgr)
        yield layout, YUV420.from_buffer(torch.from_numpy(buf.copy()), layout), bgr
        pitched = np.full((h * 3 // 2, 64), 0xEE, np.uint8)           # rows padded to a 64-byte pitch
        if layout in ("NV12", "NV21"):
            pitched[:, :w] = buf
        else:                              # chroma rows at half the luma pitch
            pitched[:h, :w] = Y
            a, b = (U, V) if layout == "I420" else (V, U)
            chroma = pitched[h:].reshape(-1)
            chroma.reshape(h, 32)[:, :w // 2] = np.concatenate([a, b])
        yield layout + "_pitched", YUV420.from_buffer(torch.from_numpy(pitched)[:, :w], layout), bgr
    # a 1088-row pitched luma surface with the chroma after the padding rows (as decoders pad 1080p)
    surf = np.full((h + 6 + h // 2, 64), 0x11, np.uint8)
    surf[:h, :w] = Y
    surf[h + 6:, :w] = np.stack([U, V], -1).reshape(h // 2, w)
    t = torch.from_numpy(surf)
    yield "nv12_padded_surface", YUV420.nv12(t[:h, :w], t[h + 6:, :w]), bgr
    # luma and interleaved chroma in separate allocations, chroma as [H/2, W/2, 2]
    yield "nv12_split", YUV420.nv12(torch.from_numpy(Y.copy()), torch.from_numpy(np.stack([U, V], -1))), bgr
    # even-offset crops of a larger frame, in every layout
    Yb, Ub, Vb = random_planes(rng, 60, 80)
    for layout in yuv.LAYOUTS:
        big = YUV420.from_buffer(torch.from_numpy(yuv.planes_to_buffer(Yb, Ub, Vb, layout)), layout)
        crop = YUV420(big.y[8:42, 14:72], big.u[4:21, 7:36], big.v[4:21, 7:36])
        yield layout + "_crop", crop, yuv.yuv_to_bgr(Yb[8:42, 14:72], Ub[4:21, 7:36], Vb[4:21, 7:36])


@pytest.mark.parametrize("name,frame,bgr", list(frames()), ids=[f[0] for f in frames()])
def test_descriptors_read_the_frame(name, frame, bgr):
    assert frame.shape == bgr.shape
    assert frame.hw("x", 0) == bgr.shape[:2]
    assert np.array_equal(yuv.yuv_to_bgr(*read_back(frame)), bgr)


def test_constructors_build_views_not_copies():
    buf = torch.zeros(48, 40, dtype=torch.uint8)
    for layout in yuv.LAYOUTS:
        f = YUV420.from_buffer(buf, layout)
        assert all(p.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr() for p in f)
    y, uv = torch.zeros(32, 40, dtype=torch.uint8), torch.zeros(16, 40, dtype=torch.uint8)
    f = YUV420.nv12(y, uv)
    assert f.y is y and f.u.untyped_storage().data_ptr() == f.v.untyped_storage().data_ptr() == uv.untyped_storage().data_ptr()


def test_constructors_reject_what_cannot_be_viewed():
    with pytest.raises(ValueError, match="layout"):
        YUV420.from_buffer(torch.zeros(48, 40, dtype=torch.uint8), "NV16")
    for shape in ((47, 40), (48, 41), (0, 40)):
        with pytest.raises(ValueError, match=r"not \[H\*3/2, W\]"):
            YUV420.from_buffer(torch.zeros(shape, dtype=torch.uint8), "NV12")
    with pytest.raises(ValueError, match="uint8"):
        YUV420.from_buffer(torch.zeros(48, 40, dtype=torch.int16), "NV12")
    wide = torch.zeros(48, 81, dtype=torch.uint8)
    with pytest.raises(ValueError, match="even pitch"):       # pitch 81: chroma rows at half of it do not exist
        YUV420.from_buffer(wide[:, :40], "I420")
    assert YUV420.from_buffer(wide[:, :40], "NV12").u.shape == (16, 20)
    with pytest.raises(ValueError, match="even pitch"):
        YUV420.from_buffer(torch.zeros(40, 48, dtype=torch.uint8).t(), "YV12")
    with pytest.raises(ValueError, match="uv must be"):
        YUV420.nv12(torch.zeros(32, 40, dtype=torch.uint8), torch.zeros(16, 20, 3, dtype=torch.uint8))


# ---- call rules ---------------------------------------------------------------------------------------------------------

class FakeCuda(torch.Tensor):
    """Stands in for a CUDA tensor of cuda:`index` on a machine without one (only the metadata the rules read)."""
    index = 0

    @property
    def is_cuda(self):
        return True

    @property
    def device(self):
        return torch.device("cuda", self.index)


def fake(shape, index=0):
    t = torch.zeros(shape, dtype=torch.uint8).as_subclass(FakeCuda)
    t.index = index
    return t


def fake_frame(h=40, w=50, index=(0, 0, 0)):
    return YUV420(fake((h, w), index[0]), fake((h // 2, w // 2), index[1]), fake((h // 2, w // 2), index[2]))


DEV = torch.device("cuda", 0)


def test_a_call_takes_one_kind_of_image():
    host, tensor = np.zeros((40, 50, 3), np.uint8), fake((40, 50, 3))
    assert images_on_device([fake_frame(), fake_frame()], DEV, "rois_images") == FRAME
    assert images_on_device([tensor], DEV, "x") is TENSOR and images_on_device([host], DEV, "x") is HOST
    with pytest.raises(ValueError, match=r"rois_images: image 2 is a host image but image 0 is a YUV420 frame.*not both"):
        images_on_device([fake_frame(), fake_frame(), host], DEV, "rois_images")
    with pytest.raises(ValueError, match=r"detect_images: image 1 is a YUV420 frame but image 0 is a CUDA tensor"):
        images_on_device([tensor, fake_frame()], DEV, "detect_images")
    with pytest.raises(ValueError, match=r"image 1 is a YUV420 frame but image 0 is a host image"):
        images_on_device([host, fake_frame()], DEV, "detect_lines_images")


@pytest.mark.parametrize("plane", [0, 1, 2])
def test_a_plane_on_another_device_or_on_the_host_is_rejected(plane):
    index = [0, 0, 0]
    index[plane] = 1
    with pytest.raises(ValueError, match=r"stream_rois_images: image 4: YUV420 plane %s is on cuda:1, the engine runs on "
                                         r"cuda:0" % "yuv"[plane]):
        on_device(fake_frame(index=tuple(index)), DEV, "stream_rois_images", 4)
    planes = list(fake_frame())
    planes[plane] = torch.zeros(tuple(planes[plane].shape), dtype=torch.uint8)
    with pytest.raises(ValueError, match="plane %s is not a CUDA tensor" % "yuv"[plane]):
        images_on_device([fake_frame(), YUV420(*planes)], DEV, "rois_images")


def test_frames_convert_to_bgr_only():
    assert on_device(fake_frame(), DEV, "x", 0, "BGR") == FRAME
    with pytest.raises(ValueError, match=r"rois_images: image 0 is a YUV420 frame, which converts to BGR; channels='RGB'"):
        images_on_device([fake_frame()], DEV, "rois_images", "RGB")


@pytest.mark.parametrize("hw", [(41, 50), (40, 51), (1, 2)])
def test_odd_sides_fail_the_plan(hw):
    h, w = hw
    with pytest.raises(ValueError, match=r"image 0 is a %dx%d YUV420 frame; 4:2:0 frames have even sides" % (h, w)):
        frontend_plan([YUV420(fake((h, w)), fake((h // 2, w // 2)), fake((h // 2, w // 2)))])


def test_malformed_planes_fail_the_plan():
    with pytest.raises(ValueError, match="image 1: YUV420 plane u is"):
        frontend_plan([fake_frame(), YUV420(fake((40, 50)), fake((20, 24)), fake((20, 25)))])
    with pytest.raises(ValueError, match="image 0: YUV420 plane v must be a 2-D uint8 tensor"):
        frontend_plan([YUV420(fake((40, 50)), fake((20, 25)), fake((20, 25, 1)))])
    with pytest.raises(ValueError, match="image 0: YUV420 plane y must be a 2-D uint8 tensor"):
        frontend_plan([YUV420(torch.zeros(40, 50), fake((20, 25)), fake((20, 25)))])


def test_a_frame_plans_as_its_bgr_image():
    for hw in ((40, 50), (1080, 1920), (2160, 3840), (1920, 1080)):
        assert frontend_plan([fake_frame(*hw)])[0] == frontend_plan([hw])[0]


def test_frame_streams_upload_the_sizes_only():
    shapes = [(1080, 1920), (720, 1280), (2160, 3840)]
    items = frontend_plan([fake_frame(*s) for s in shapes])
    lay = stream_layout(items, shapes, sources=False)
    assert lay.total == 28 * 3 and lay.offsets is None
    buf = np.full(lay.total, 0xAB, np.uint8)
    stream_pack(buf, lay, StreamBatch([0, 1, 2], items, [fake_frame(*s) for s in shapes], (600, 1067)))
    assert np.array_equal(buf[:24].view(np.int32), np.array([p.blob for p in items], np.int32).ravel())
