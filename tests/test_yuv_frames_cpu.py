"""CPU: YUV420Frame, the FearFrameYUV420 records it builds, and FEARMultiTracker's checks of YUV frames."""
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib

CFG = fb.FEAR_XS_TRACKER_KWARGS
LAYOUTS = ("nv12", "pitched", "planes", "i420", "roi")
RGB = np.zeros((64, 80, 3), np.uint8)


def split_i420(i420: np.ndarray):
    """The y (H, W), u and v (H/2, W/2) planes of a (3H/2, W) array in cv2's I420 layout."""
    h, w = 2 * i420.shape[0] // 3, i420.shape[1]
    flat, q = i420.reshape(-1), h * w // 4
    return flat[:h * w].reshape(h, w), flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2,
                                                                                                                w // 2)


def yuv_frame(i420: np.ndarray, layout: str, device="cuda") -> fb.YUV420Frame:
    """The frame held by ``i420`` (cv2's I420 layout) as a YUV420Frame on ``device``, freshly allocated, laid out as
    contiguous NV12, NV12 with a row pitch of 512 bytes or more, NV12 with Y and UV in separate allocations, I420, or
    an even-offset region of interest of a larger NV12 surface.  Bytes outside the frame are filled with 0xA5."""
    y, u, v = split_i420(i420)
    h, w = y.shape
    uv = np.stack([u, v], -1).reshape(h // 2, w)
    nv12 = np.concatenate([y, uv])

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device)

    if layout == "nv12":
        return fb.YUV420Frame.nv12(dev(nv12))
    if layout == "pitched":
        surface = torch.full((nv12.shape[0], 512 * (w // 512 + 1)), 0xA5, dtype=torch.uint8, device=device)
        surface[:, :w] = dev(nv12)
        return fb.YUV420Frame.nv12(surface[:, :w])
    if layout == "planes":
        luma, chroma = dev(y), dev(uv)
        return fb.YUV420Frame(luma, chroma[:, 0::2], chroma[:, 1::2])
    if layout == "i420":
        return fb.YUV420Frame.i420(dev(i420))
    if layout == "roi":  # the frame at luma offset (2, 4) of an NV12 surface of (H + 6, W + 10)
        hb = h + 6
        big = torch.full((hb * 3 // 2, w + 10), 0xA5, dtype=torch.uint8, device=device)
        big[2:2 + h, 4:4 + w] = dev(y)
        big[hb + 1:hb + 1 + h // 2, 4:4 + w] = dev(uv)
        c = big[hb + 1:hb + 1 + h // 2]
        return fb.YUV420Frame(big[2:2 + h, 4:4 + w], c[:, 4:4 + w:2], c[:, 5:5 + w:2])
    raise ValueError(layout)


def _tracker():
    net = fb.FEARNet(**fb.FEAR_XS_MODEL_KWARGS).eval()
    return fb.FEARMultiTracker(net, cuda_id="cpu", max_targets=4, **CFG)


def test_yuv420_record_is_64_bytes():
    assert _lib.YUV420_DTYPE.itemsize == 64
    assert _lib.YUV420_DTYPE.names == ("y", "u", "v", "y_row_stride", "y_pixel_stride", "uv_row_stride",
                                       "uv_pixel_stride", "H", "W")


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("hw", [(2, 2), (6, 10), (90, 334), (256, 480)])
def test_record_addresses_the_planes(layout, hw):
    """Reading each plane's storage through the record's address and strides gives the plane's bytes."""
    h, w = hw
    i420 = np.random.default_rng(h * w).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    f = yuv_frame(i420, layout, device="cpu")
    assert f.shape == (h, w, 3)
    rec = np.array([f.record()], dtype=_lib.YUV420_DTYPE)[0]
    assert (int(rec["H"]), int(rec["W"])) == (h, w)
    strides = {"y": (rec["y_row_stride"], rec["y_pixel_stride"]), "u": (rec["uv_row_stride"], rec["uv_pixel_stride"]),
               "v": (rec["uv_row_stride"], rec["uv_pixel_stride"])}
    for name, want in zip("yuv", split_i420(i420)):
        plane = getattr(f, name)
        storage = np.frombuffer(bytes(plane.untyped_storage()), dtype=np.uint8)
        off = int(rec[name]) - plane.untyped_storage().data_ptr()
        rs, ps = (int(s) for s in strides[name])
        r, c = np.meshgrid(np.arange(want.shape[0]), np.arange(want.shape[1]), indexing="ij")
        assert np.array_equal(storage[off + r * rs + c * ps], want), (layout, name)
    if layout == "pitched":
        assert rec["y_row_stride"] >= 512 and rec["uv_pixel_stride"] == 2 and int(rec["v"]) - int(rec["u"]) == 1


def test_nv12_and_i420_records_follow_the_documented_layouts():
    h, w, p = 6, 10, 512
    surface = torch.zeros(h * 3 // 2, p, dtype=torch.uint8)
    b = surface.data_ptr()
    assert fb.YUV420Frame.nv12(surface[:, :w]).record() == (b, b + h * p, b + h * p + 1, p, 1, p, 2, h, w)
    packed = torch.zeros(h * 3 // 2, w, dtype=torch.uint8)
    b = packed.data_ptr()
    q = h * w // 4
    assert fb.YUV420Frame.i420(packed).record() == (b, b + h * w, b + h * w + q, w, 1, w // 2, 1, h, w)


def _planes(h, w, dtype=torch.uint8):
    return torch.zeros(h, w, dtype=dtype), torch.zeros(h // 2, w // 2, dtype=dtype), torch.zeros(h // 2, w // 2,
                                                                                                   dtype=dtype)


BAD_CONSTRUCTIONS = {
    "odd H": lambda: fb.YUV420Frame(torch.zeros(63, 80, dtype=torch.uint8), *_planes(62, 80)[1:]),
    "odd W": lambda: fb.YUV420Frame(torch.zeros(64, 81, dtype=torch.uint8), *_planes(64, 80)[1:]),
    "odd W nv12": lambda: fb.YUV420Frame.nv12(torch.zeros(96, 81, dtype=torch.uint8)),
    "odd W i420": lambda: fb.YUV420Frame.i420(torch.zeros(96, 81, dtype=torch.uint8)),
    "H < 2": lambda: fb.YUV420Frame.nv12(torch.zeros(0, 80, dtype=torch.uint8)),
    "rows not 3H/2": lambda: fb.YUV420Frame.nv12(torch.zeros(97, 80, dtype=torch.uint8)),
    "chroma shape": lambda: fb.YUV420Frame(*_planes(64, 80)[:2], torch.zeros(32, 41, dtype=torch.uint8)),
    "chroma full size": lambda: fb.YUV420Frame(*_planes(64, 80)[:1], *_planes(128, 160)[1:]),
    "luma 3-D": lambda: fb.YUV420Frame(torch.zeros(64, 80, 1, dtype=torch.uint8), *_planes(64, 80)[1:]),
    "u, v strides": lambda: fb.YUV420Frame(_planes(64, 80)[0], torch.zeros(32, 80, dtype=torch.uint8)[:, 0::2],
                                           torch.zeros(32, 40, dtype=torch.uint8)),
    "float planes": lambda: fb.YUV420Frame(*_planes(64, 80, torch.float32)),
    "int16 luma": lambda: fb.YUV420Frame(torch.zeros(64, 80, dtype=torch.int16), *_planes(64, 80)[1:]),
    "int16 nv12": lambda: fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.int16)),
    "numpy planes": lambda: fb.YUV420Frame(*(p.numpy() for p in _planes(64, 80))),
    "i420 not contiguous": lambda: fb.YUV420Frame.i420(torch.zeros(96, 160, dtype=torch.uint8)[:, ::2]),
    "CPU planes": lambda: fb.YUV420Frame(*_planes(64, 80)),
    "CPU nv12": lambda: fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8)),
    "YUV then RGB": lambda: [fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8)), RGB],
    "RGB then YUV": lambda: [RGB, fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8))],
    "tensor then YUV": lambda: [torch.zeros(64, 80, 3, dtype=torch.uint8),
                                fb.YUV420Frame.i420(torch.zeros(96, 80, dtype=torch.uint8))],
}


@pytest.mark.parametrize("what", list(BAD_CONSTRUCTIONS))
def test_bad_yuv_frames_are_refused_before_device_calls(what):
    """Malformed frames are refused by YUV420Frame's constructors, well-formed ones in host memory or mixed with RGB
    frames by the tracker; either way with ValueError from add and update, with and without a live target, before
    any device call (there is no device here)."""
    make = BAD_CONSTRUCTIONS[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[10, 10, 20, 20]])
    with pytest.raises(ValueError):
        trk.update(make())
    trk._ids, trk._streams = np.array([0]), np.array([0])  # a live target: update reaches the frame checks the same way
    with pytest.raises(ValueError):
        trk.update(make())
