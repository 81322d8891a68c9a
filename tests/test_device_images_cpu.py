"""CPU: the host side of photos already in device memory.  ctpn_resize_linear_u8_strided rejects every bad descriptor
before any CUDA call; the engine's descriptor builder, read back through the same byte arithmetic as the kernel, gives
the BGR image for every layout a caller will have; and the rules of the raw-photo calls -- all-host or all-device, one
channel order per call, RGB host images flipped in the packing copy -- hold without a device."""
import ctypes as C

import numpy as np
import pytest
import torch

from ctpn_b200 import _native as N
from ctpn_b200.engine import (StreamBatch, check_channels, frontend_plan, images_on_device, on_device, stream_layout,
                              stream_pack, strided_descriptor, tensor_descriptor)
from oracle import resize as R

FAKE = 0x10000        # a non-null "device" address: validation fails before anything dereferences it


# ---- ctpn_resize_linear_u8_strided: validation before any CUDA call -------------------------------------------------

def descriptors():
    """Three images: a dense 100 x 60 HWC image, the 30 x 50 RGB top-left crop of a 64-pixel-wide frame read from channel 2
    backwards, and a 64 x 96 CHW image (planar); each in an allocation of its own whose first and last bytes it touches."""
    return dict(src=np.array([FAKE, FAKE + (1 << 24), FAKE + (1 << 25)], np.uint64),
                nbytes=np.array([100 * 60 * 3, 29 * 64 * 3 + 50 * 3, 3 * 64 * 96], np.uint64),
                offs=np.array([0, 2, 0], np.int64),
                strides=np.array([[180, 3, 1], [64 * 3, 3, -1], [96, 1, 64 * 96]], np.int64),
                hw=np.array([[100, 60], [30, 50], [64, 96]], np.int32),
                fxy=np.array([[0.2, 0.2], [0.5, 0.5], [1.0, 1.0]], np.float64),
                dst=np.array([R.out_size(100, 60, 0.2, 0.2), R.out_size(30, 50, 0.5, 0.5), R.out_size(64, 96, 1.0, 1.0)],
                             np.int32),
                B=3, H=64, W=96)


def call(d, dst=C.c_void_p(FAKE), null=()):
    a = {k: (None if k in null else N.ptr(np.ascontiguousarray(d[k]))) for k in ("src", "nbytes", "offs", "strides", "hw", "fxy",
                                                                                  "dst")}
    rc = N.lib.ctpn_resize_linear_u8_strided(a["src"], a["nbytes"], a["offs"], a["strides"], a["hw"], a["fxy"], a["dst"], d["B"],
                                             dst, d["H"], d["W"], None)
    return rc, N.last_error()


def test_valid_descriptors_stop_at_the_device_query():
    if torch.cuda.is_available():
        pytest.skip("the call would launch on the fake pointers; only meaningful without a GPU")
    rc, msg = call(descriptors())
    assert rc == N.ERR_NO_DEVICE, msg


@pytest.mark.parametrize("B", [0, -1, 65])
def test_batch_size_within_1_to_64(B):
    d = descriptors()
    d["B"] = B
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "B = %d" % B in msg


def test_null_pointers_are_invalid():
    d = descriptors()
    rc, msg = call(d, dst=None)
    assert rc == N.ERR_INVALID and "null" in msg
    for name in ("src", "nbytes", "offs", "strides", "hw", "fxy", "dst"):
        rc, msg = call(d, null=(name,))
        assert rc == N.ERR_INVALID and "null" in msg, name
    d["src"][1] = 0
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1" in msg and "null" in msg


@pytest.mark.parametrize("b", [0, 1, 2])
def test_the_box_must_end_inside_the_allocation(b):
    d = descriptors()
    d["nbytes"][b] -= 1                    # each image's highest byte is the last byte of its allocation
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image %d" % b in msg and "outside" in msg


@pytest.mark.parametrize("b", [0, 1, 2])
def test_the_box_must_start_inside_the_allocation(b):
    d = descriptors()
    d["offs"][b] -= 1                      # image 1 reaches byte 0 through its negative channel stride
    d["nbytes"][b] += 1                    # the highest byte alone would still fit
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image %d" % b in msg and "outside" in msg


def test_negative_strides_reach_below_the_offset():
    d = descriptors()
    d["offs"][0] = 99 * 180 + 59 * 3 + 2   # image 0 read bottom-up, right to left, RGB: every stride negative
    d["strides"][0] = [-180, -3, -1]
    d["nbytes"][0] = 100 * 60 * 3
    rc, msg = call(d)
    assert "image 0" not in msg, msg
    d["offs"][0] -= 1
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "outside" in msg


def test_zero_strides_broadcast():
    d = descriptors()
    d["strides"][0] = [0, 0, 0]            # one byte, read everywhere
    d["nbytes"][0] = 1
    rc, msg = call(d)
    assert "image 0" not in msg, msg
    d["offs"][0] = 1
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "outside" in msg
    d["offs"][0] = 0
    d["strides"][0] = [3, 0, 1]            # a column broadcast of a 100-pixel column: 300 bytes
    d["nbytes"][0] = 300
    rc, msg = call(d)
    assert "image 0" not in msg, msg
    d["nbytes"][0] = 299
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg


@pytest.mark.parametrize("stride", [1 << 62, -(1 << 62), (1 << 63) - 1])
def test_the_extent_arithmetic_does_not_wrap(stride):
    d = descriptors()
    d["strides"][0][0] = stride            # 99 rows of it: far outside any int64
    d["nbytes"][0] = (1 << 64) - 1
    d["offs"][0] = (1 << 63) - 1 if stride < 0 else 0
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "outside" in msg
    d = descriptors()
    d["offs"][2] = (1 << 63) - 1           # offset alone at the end of the int64 range
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg


@pytest.mark.parametrize("axis", [1, 2])
def test_column_and_channel_strides_fit_32_bits(axis):
    d = descriptors()
    d["strides"][0][axis] = 1 << 31
    d["nbytes"][0] = 1 << 40
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "32-bit" in msg


def test_sizes_scales_dst_and_canvas():
    d = descriptors()
    d["hw"][1] = [0, 50]
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 1" in msg and "source size" in msg
    d = descriptors()
    d["fxy"][2] = [0.0, 1.0]
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "scale" in msg
    d = descriptors()
    d["dst"][0] = [d["dst"][0][0] + 1, d["dst"][0][1]]       # not what cv2 would produce
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 0" in msg and "cv2 would produce" in msg
    d = descriptors()
    d["W"] = 95                            # image 2's 96 columns do not fit
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "image 2" in msg and "canvas" in msg
    d = descriptors()
    d["H"] = 0
    rc, msg = call(d)
    assert rc == N.ERR_INVALID and "canvas" in msg


# ---- the descriptor builder --------------------------------------------------------------------------------------------

def read_back(desc, h, w, storage):
    """The h x w x 3 image the kernel reads through a descriptor: sample (y, x, c) at byte offset + y*rs + x*cs + c*ks of the
    allocation (here a host copy of the storage bytes)."""
    _, nbytes, off, (rs, cs, ks) = desc
    assert len(storage) == nbytes
    y, x, c = np.meshgrid(np.arange(h), np.arange(w), np.arange(3), indexing="ij")
    idx = off + y * rs + x * cs + c * ks
    assert idx.min() >= 0 and idx.max() < nbytes
    return storage[idx]


def storage_bytes(t):
    st = t.untyped_storage()
    return torch.empty(0, dtype=torch.uint8).set_(st, 0, (st.nbytes(),), (1,)).numpy().copy()


def layouts():
    rng = np.random.default_rng(3)
    bgr = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    frame = torch.from_numpy(rng.integers(0, 256, (60, 80, 3), dtype=np.uint8))
    chw = torch.from_numpy(np.ascontiguousarray(bgr.transpose(2, 0, 1)))
    rgb_chw = torch.from_numpy(np.ascontiguousarray(bgr[:, :, ::-1].transpose(2, 0, 1)))
    yield "hwc", torch.from_numpy(bgr.copy()), "BGR", bgr
    yield "rgb_hwc", torch.from_numpy(np.ascontiguousarray(bgr[:, :, ::-1])), "RGB", bgr
    yield "crop", frame[11:48, 20:73], "BGR", frame.numpy()[11:48, 20:73]
    yield "rgb_crop", frame[11:48, 20:73], "RGB", frame.numpy()[11:48, 20:73, ::-1]
    yield "chw", chw.permute(1, 2, 0), "BGR", bgr
    yield "rgb_chw", rgb_chw.permute(1, 2, 0), "RGB", bgr
    yield "rgb_chw_crop", rgb_chw[:, 3:30, 5:50].permute(1, 2, 0), "RGB", bgr[3:30, 5:50]
    px = torch.tensor([[[10, 20, 30]]], dtype=torch.uint8)
    yield "broadcast", px.expand(37, 53, 3), "BGR", np.broadcast_to(px.numpy(), (37, 53, 3))
    row = torch.from_numpy(bgr[:1].copy())
    yield "rgb_broadcast_rows", row.expand(37, 53, 3), "RGB", np.broadcast_to(bgr[:1, :, ::-1], (37, 53, 3))


@pytest.mark.parametrize("name,t,channels,want", list(layouts()), ids=[x[0] for x in layouts()])
def test_descriptor_reads_the_bgr_image(name, t, channels, want):
    desc = tensor_descriptor(t, channels)
    assert desc[0] == t.untyped_storage().data_ptr() and desc[1] == t.untyped_storage().nbytes()
    h, w = t.shape[:2]
    assert np.array_equal(read_back(desc, h, w, storage_bytes(t)), want)


def test_strided_descriptor_from_metadata():
    assert strided_descriptor(0x1000, 300, 7, (30, 3, 1)) == (0x1000, 300, 7, (30, 3, 1))
    assert strided_descriptor(0x1000, 300, 7, (30, 3, 1), "RGB") == (0x1000, 300, 9, (30, 3, -1))
    assert strided_descriptor(0x2000, 3 * 40, 0, (8, 1, 40), "RGB") == (0x2000, 120, 80, (8, 1, -40))   # planar CHW
    assert strided_descriptor(0x2000, 3, 0, (0, 0, 1), "RGB") == (0x2000, 3, 2, (0, 0, -1))
    with pytest.raises(ValueError, match="channels"):
        strided_descriptor(0x1000, 300, 0, (30, 3, 1), "bgr")


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


def fake(h=40, w=50, index=0):
    t = torch.zeros(h, w, 3, dtype=torch.uint8).as_subclass(FakeCuda)
    t.index = index
    return t


DEV = torch.device("cuda", 0)


def test_a_call_is_all_host_or_all_device():
    host = np.zeros((40, 50, 3), np.uint8)
    assert images_on_device([fake(), fake()], DEV, "rois_images") is True
    assert images_on_device([host, torch.zeros(40, 50, 3, dtype=torch.uint8)], DEV, "rois_images") is False   # CPU tensors are host images
    assert images_on_device([], DEV, "rois_images") is False
    with pytest.raises(ValueError, match=r"rois_images: image 2 is a host image but image 0 is a CUDA tensor"):
        images_on_device([fake(), fake(), host], DEV, "rois_images")
    with pytest.raises(ValueError, match=r"detect_images: image 1 is a CUDA tensor but image 0 is a host image"):
        images_on_device([host, fake(), host], DEV, "detect_images")


def test_a_tensor_on_another_device_is_rejected():
    assert on_device(fake(), DEV, "x", 0)
    with pytest.raises(ValueError, match=r"stream_rois_images: image 4 is on cuda:1, the engine runs on cuda:0"):
        on_device(fake(index=1), DEV, "stream_rois_images", 4)
    with pytest.raises(ValueError, match="image 1 is on cuda:1"):
        images_on_device([fake(), fake(index=1)], DEV, "rois_images")


def test_device_tensors_of_another_dtype_or_shape_fail_the_plan():
    bad = torch.zeros(40, 50, 4, dtype=torch.uint8).as_subclass(FakeCuda)
    with pytest.raises(ValueError, match="image 0 must be HxWx3 uint8"):
        frontend_plan([bad])
    bad = torch.zeros(40, 50, 3, dtype=torch.float32).as_subclass(FakeCuda)
    with pytest.raises(ValueError, match="image 0 must be HxWx3 uint8"):
        frontend_plan([bad])
    assert frontend_plan([fake()])[0] == frontend_plan([(40, 50)])[0]


@pytest.mark.parametrize("channels", ["bgr", "RGBA", None, ""])
def test_channels_is_bgr_or_rgb(channels):
    check_channels("BGR", "x")
    check_channels("RGB", "x")
    with pytest.raises(ValueError, match="stream_images: channels must be 'BGR' or 'RGB'"):
        check_channels(channels, "stream_images")


def test_device_streams_upload_the_sizes_only():
    items = frontend_plan([(3024, 4032), (600, 800), (1080, 1920)])
    lay = stream_layout(items, [(3024, 4032), (600, 800), (1080, 1920)], sources=False)
    assert lay.total == 28 * 3 and lay.sizes_at == 0 and lay.maps is None and lay.offsets is None
    buf = np.full(lay.total, 0xAB, np.uint8)
    stream_pack(buf, lay, StreamBatch([0, 1, 2], items, [fake(), fake(), fake()], (600, 1200)))
    blobs = np.array([p.blob for p in items], np.int32)
    assert np.array_equal(buf[:24].view(np.int32), blobs.ravel())
    assert np.array_equal(buf[24:48].view(np.int32), (blobs >> 4).ravel())


@pytest.mark.parametrize("compact", [False, True])
def test_rgb_host_images_are_flipped_by_the_packing_copy(compact):
    rng = np.random.default_rng(5)
    shapes = [(2000, 2200), (300, 400)]    # a strong downscale, sent as the rows it reads, and a whole image
    ims = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    items = frontend_plan(ims)
    assert (items[0].rows is not None) and items[1].rows is None
    lay = stream_layout(items, shapes, compact)
    batch = StreamBatch([0, 1], items, ims, (600, 600))
    want = np.zeros(lay.total, np.uint8)
    stream_pack(want, lay, batch._replace(images=[np.ascontiguousarray(im[:, :, ::-1]) for im in ims]))
    got = np.zeros(lay.total, np.uint8)
    stream_pack(got, lay, batch, "RGB")
    assert np.array_equal(got, want)
