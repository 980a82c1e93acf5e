"""CPU: YUV422Frame and YUV444Frame, the FearFrameYCbCr records every YUV frame builds, and image_ops.yuv_to_rgb, the
numpy restatement of the kernels' conversion at every chroma subsampling that the GPU tests compare against.

The restatement is pinned to cv2.cvtColor's YUY2 / UYVY / YVYU conversion on all 2^24 (Y, U, V) triples, and to
yuv420_to_rgb (itself pinned by tests/test_yuv_formats_cpu.py) for every format: at shifts (1, 1) directly, and at
4:2:2 / 4:4:4 on frames whose chroma repeats 4:2:0 chroma."""
import itertools

import cv2
import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from tests.test_yuv_formats_cpu import FORMATS
from tests.test_yuv_frames_cpu import RGB, _tracker

LAYOUTS_422 = ("yuyv", "yuyv_pitched", "uyvy", "yvyu", "nv16", "nv16_pitched", "i422", "planes422", "roi422")
LAYOUTS_444 = ("i444", "i444_pitched", "i444_msb_pitched", "planes444", "roi444")
PACKED = {"yuyv": ((0, 2), (1, 4), (3, 4)), "uyvy": ((1, 2), (0, 4), (2, 4)), "yvyu": ((0, 2), (3, 4), (1, 4))}
CV2_PACKED = {"yuyv": cv2.COLOR_YUV2RGB_YUY2, "uyvy": cv2.COLOR_YUV2RGB_UYVY, "yvyu": cv2.COLOR_YUV2RGB_YVYU}


def layout_msb(layout: str, bits: int) -> bool:
    """Whether ``layout`` holds 10 / 12-bit samples in the high bits: Y210 / P210 (the packed and NV16 layouts and the
    regions of interest cut from them) and NVDEC's 16-bit 4:4:4; yuv422p10le / yuv444p10le are LSB-aligned."""
    return bits > 8 and (layout.split("_")[0] in (*PACKED, "nv16", "roi422", "roi444") or "msb" in layout)


def ycbcr_frame(y, u, v, layout: str, bits: int = 8, device="cuda", rng=None, **fmt):
    """Code planes (Y (H, W); U, V (H, W/2) for a 4:2:2 layout, (H, W) for a 4:4:4 one) as a freshly allocated
    YUV422Frame / YUV444Frame on ``device``, through the constructor of ``layout``:

        yuyv, uyvy, yvyu     packed (H, 2W) rows (Y210 at 10 / 12 bits); *_pitched: with a row pitch
        nv16                 (2H, W): luma rows, then interleaved (U, V) rows (P210 at 10 / 12 bits)
        i422                 contiguous (2H, W) planes one after another (yuv422p10le at 10 / 12 bits)
        planes422            YUV422Frame(y, u, v) of three allocations
        roi422               the frame at row 3, column 2 of a larger YUYV / Y210 surface: an odd row offset
        i444                 (3H, W) planes one after another (yuv444p10le); *_pitched with a row pitch; i444_msb_* the
                             16-bit NVDEC surface (MSB-aligned)
        planes444            YUV444Frame(y, u, v) of three allocations
        roi444               the frame at (2, 3) of three planes of a larger surface: an odd column offset

    Samples hold the codes aligned as the layout stores them (``layout_msb``); with ``rng`` the bits the reader masks
    hold noise.  Samples outside the frame are 0xA5 / 0xA5A5."""
    wide = bits > 8
    msb = layout_msb(layout, bits)
    rng = rng if rng is not None else np.random.default_rng(0)

    def samples(c):
        c = np.asarray(c).astype(np.int64)
        if not wide:
            return c.astype(np.uint8)
        noise = rng.integers(0, 1 << (16 - bits), c.shape)
        return ((c << (16 - bits)) | noise if msb else c | (noise << bits)).astype(np.uint16)

    Y, U, V = samples(y), samples(u), samples(v)
    h, w = Y.shape
    dt = np.uint16 if wide else np.uint8
    fill = 0xA5A5 if wide else 0xA5

    def dev(a):
        a = np.ascontiguousarray(a, dtype=dt)
        return torch.from_numpy(a.view(np.int16)).view(torch.uint16).to(device) if wide else \
            torch.from_numpy(a).to(device)

    def pitched(a, rows=None, r0=0, c0=0, pad=40):  # a at (r0, c0) of a 0xA5-filled surface, as a view
        big = np.full((a.shape[0] + r0 + 5, a.shape[1] + c0 + pad), fill, dt)
        big[r0:r0 + a.shape[0], c0:c0 + a.shape[1]] = a
        return dev(big)[r0:r0 + a.shape[0], c0:c0 + a.shape[1]]

    base = layout.split("_")[0]
    kw = dict(fmt, bits=bits)
    if base in PACKED or base == "roi422":
        order = "yuyv" if base == "roi422" else base
        (yo, ys), (uo, us), (vo, vs) = PACKED[order]
        row = np.empty((h, 2 * w), dt)
        row[:, yo::ys], row[:, uo::us], row[:, vo::vs] = Y, U, V
        make = getattr(fb.YUV422Frame, order)
        if base == "roi422":
            return make(pitched(row, r0=3, c0=4), **kw)
        return make(pitched(row) if layout.endswith("pitched") else dev(row), **kw)
    if base == "nv16":
        nv = np.concatenate([Y, np.stack([U, V], -1).reshape(h, w)])
        return fb.YUV422Frame.nv16(pitched(nv) if layout.endswith("pitched") else dev(nv), **kw)
    if base in ("i422", "i444"):
        flat = np.concatenate([Y.reshape(-1), U.reshape(-1), V.reshape(-1)])
        rows = flat.reshape(-1, w)
        if base == "i422":
            return fb.YUV422Frame.i422(dev(rows), **kw)
        return fb.YUV444Frame.i444(pitched(rows) if layout.endswith("pitched") else dev(rows), msb=msb, **kw)
    if base in ("planes422", "planes444"):
        cls = fb.YUV422Frame if base == "planes422" else fb.YUV444Frame
        return cls(dev(Y), dev(U), dev(V), msb=msb, **kw)
    if base == "roi444":
        big = np.full((3, h + 6, w + 9), fill, dt)
        big[0, 2:2 + h, 3:3 + w], big[1, 2:2 + h, 3:3 + w], big[2, 2:2 + h, 3:3 + w] = Y, U, V
        t = dev(big)
        return fb.YUV444Frame(t[0, 2:2 + h, 3:3 + w], t[1, 2:2 + h, 3:3 + w], t[2, 2:2 + h, 3:3 + w], msb=msb, **kw)
    raise ValueError(layout)


def oracle(y, u, v, chroma_shift, matrix="bt601", full_range=False, bits=8) -> np.ndarray:
    """image_ops.yuv_to_rgb of code planes."""
    return image_ops.yuv_to_rgb(y, u, v, matrix, full_range, bits, 0, chroma_shift)


def test_ycbcr_record_is_88_bytes():
    assert _lib.YCBCR_DTYPE.itemsize == 88
    assert _lib.YCBCR_DTYPE.names == ("y", "u", "v", "y_row_stride", "y_pixel_stride", "uv_row_stride",
                                      "uv_pixel_stride", "H", "W", "matrix", "full_range", "bits", "shift",
                                      "chroma_shift_x", "chroma_shift_y")


def test_new_symbols_are_exported():
    assert fb.YUV422Frame.CHROMA_SHIFT == (1, 0) and fb.YUV444Frame.CHROMA_SHIFT == (0, 0)
    assert fb.YUV420Frame.CHROMA_SHIFT == (1, 1)
    assert callable(image_ops.yuv_to_rgb)
    for name in ("fear_crop_targets_ycbcr_u8", "fear_advance_targets_ycbcr", "fear_frame_sums_ycbcr_u8"):
        assert name in _lib.exported_symbols()


# ---------------------------------------------------------------------------------------------------- records
def _read_back(f, want_planes):
    """Read each plane through the frame's FearFrameYCbCr record (address and byte strides into its storage) and
    compare with the sample planes it should hold; returns the record."""
    rec = np.array([f.ycbcr_record()], dtype=_lib.YCBCR_DTYPE)[0]
    assert (int(rec["H"]), int(rec["W"])) == f.shape[:2]
    strides = {"y": (rec["y_row_stride"], rec["y_pixel_stride"]), "u": (rec["uv_row_stride"], rec["uv_pixel_stride"]),
               "v": (rec["uv_row_stride"], rec["uv_pixel_stride"])}
    for name, want in zip("yuv", want_planes):
        plane = getattr(f, name)
        storage = np.frombuffer(bytes(plane.untyped_storage()), dtype=np.uint8)
        off = int(rec[name]) - plane.untyped_storage().data_ptr()
        rs, ps = (int(s) for s in strides[name])
        r, c = np.meshgrid(np.arange(want.shape[0]), np.arange(want.shape[1]), indexing="ij")
        at = off + r * rs + c * ps
        got = storage[at] if f.bits == 8 else storage[at] | (storage[at + 1].astype(np.uint16) << 8)
        code = got if f.bits == 8 else (got.astype(np.int64) >> f.shift) & ((1 << f.bits) - 1)
        assert np.array_equal(code, want), name
    return rec


@pytest.mark.parametrize("layout", LAYOUTS_422 + LAYOUTS_444)
@pytest.mark.parametrize("hw", [(1, 2), (3, 6), (2, 5), (45, 334)])
@pytest.mark.parametrize("bits", [8, 10, 12])
def test_record_addresses_the_planes(layout, hw, bits):
    """Contiguous, pitched and region-of-interest inputs of every constructor: reading the storage through the record
    gives the codes, and the format and chroma shifts are the frame's.  An odd W is rounded up to even at 4:2:2."""
    h, w = hw
    sx, sy = (1, 0) if layout in LAYOUTS_422 else (0, 0)
    w += w % 2 if sx else 0
    rng = np.random.default_rng(h * w + bits)
    planes = [rng.integers(0, 1 << bits, s) for s in ((h, w), (h, w >> sx), (h, w >> sx))]
    f = ycbcr_frame(*planes, layout, bits, device="cpu", rng=rng, matrix="bt709", full_range=True)
    assert f.shape == (h, w, 3)
    rec = _read_back(f, planes)
    shift = 16 - bits if layout_msb(layout, bits) else 0
    assert tuple(int(rec[k]) for k in ("matrix", "full_range", "bits", "shift", "chroma_shift_x", "chroma_shift_y")) \
        == (1, 1, bits, shift, sx, sy)


def test_records_follow_the_documented_layouts():
    """The records of include/fear_b200.h's FearFrameYCbCr table, for pitch P bytes at address b."""
    h, w, p = 5, 6, 64
    s8 = torch.zeros(3 * h, p, dtype=torch.uint8)
    s16 = torch.zeros(3 * h, p // 2, dtype=torch.uint16)
    b, b16 = s8.data_ptr(), s16.data_ptr()
    fmt = (h, w, 0, 0, 8, 0)
    assert fb.YUV422Frame.yuyv(s8[:h, :2 * w]).ycbcr_record() == (b, b + 1, b + 3, p, 2, p, 4, *fmt, 1, 0)
    assert fb.YUV422Frame.uyvy(s8[:h, :2 * w]).ycbcr_record() == (b + 1, b, b + 2, p, 2, p, 4, *fmt, 1, 0)
    assert fb.YUV422Frame.yvyu(s8[:h, :2 * w]).ycbcr_record() == (b, b + 3, b + 1, p, 2, p, 4, *fmt, 1, 0)
    assert fb.YUV422Frame.yuyv(s16[:h, :2 * w], bits=10).ycbcr_record() == \
        (b16, b16 + 2, b16 + 6, p, 4, p, 8, h, w, 0, 0, 10, 6, 1, 0)
    assert fb.YUV422Frame.nv16(s8[:2 * h, :w]).ycbcr_record() == \
        (b, b + h * p, b + h * p + 1, p, 1, p, 2, *fmt, 1, 0)
    assert fb.YUV422Frame.nv16(s16[:2 * h, :w], bits=12).ycbcr_record() == \
        (b16, b16 + h * p, b16 + h * p + 2, p, 2, p, 4, h, w, 0, 0, 12, 4, 1, 0)
    i422 = torch.zeros(2 * h, w, dtype=torch.uint8)
    b, hw = i422.data_ptr(), h * w
    assert fb.YUV422Frame.i422(i422).ycbcr_record() == (b, b + hw, b + hw + hw // 2, w, 1, w // 2, 1, *fmt, 1, 0)
    i422 = torch.zeros(2 * h, w, dtype=torch.uint16)
    b = i422.data_ptr()
    assert fb.YUV422Frame.i422(i422, bits=10).ycbcr_record() == \
        (b, b + 2 * hw, b + 3 * hw, 2 * w, 2, w, 2, h, w, 0, 0, 10, 0, 1, 0)
    b, b16 = s8.data_ptr(), s16.data_ptr()
    assert fb.YUV444Frame.i444(s8[:, :w], matrix="bt2020").ycbcr_record() == \
        (b, b + h * p, b + 2 * h * p, p, 1, p, 1, h, w, 2, 0, 8, 0, 0, 0)
    assert fb.YUV444Frame.i444(s16[:, :w], msb=True, bits=10).ycbcr_record() == \
        (b16, b16 + h * p, b16 + 2 * h * p, p, 2, p, 2, h, w, 0, 0, 10, 6, 0, 0)
    assert fb.YUV444Frame.i444(s16[:, :w], bits=12).ycbcr_record()[12] == 0


def test_yuv420_ycbcr_record_is_its_yuv_record_with_shifts_1_1():
    for f in (fb.YUV420Frame.nv12(torch.zeros(96, 80, dtype=torch.uint8)),
              fb.YUV420Frame.i420(torch.zeros(96, 80, dtype=torch.uint16), matrix="bt709", bits=10)):
        assert f.ycbcr_record() == f.yuv_record() + (1, 1)


def _u8(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


def _u16(*shape):
    return torch.zeros(*shape, dtype=torch.uint16)


BAD_FRAMES = {
    "422 odd W": lambda: fb.YUV422Frame(_u8(4, 7), _u8(4, 3), _u8(4, 3)),
    "422 chroma rows halved": lambda: fb.YUV422Frame(_u8(4, 8), _u8(2, 4), _u8(2, 4)),
    "422 chroma full width": lambda: fb.YUV422Frame(_u8(4, 8), _u8(4, 8), _u8(4, 8)),
    "422 u, v strides": lambda: fb.YUV422Frame(_u8(4, 8), _u8(4, 8)[:, 0::2], _u8(4, 4)),
    "422 negative stride": lambda: fb.YUV422Frame(_u8(4, 8), _u8(4, 4).flip(1), _u8(4, 4).flip(1)),
    "422 W = 0": lambda: fb.YUV422Frame(_u8(4, 0), _u8(4, 0), _u8(4, 0)),
    "yuyv width not 4k": lambda: fb.YUV422Frame.yuyv(_u8(4, 14)),
    "yuyv 3-D": lambda: fb.YUV422Frame.yuyv(_u8(4, 8, 2)),
    "yuyv float": lambda: fb.YUV422Frame.yuyv(torch.zeros(4, 16)),
    "uyvy uint16 at 8 bits": lambda: fb.YUV422Frame.uyvy(_u16(4, 16)),
    "y210 uint8": lambda: fb.YUV422Frame.yuyv(_u8(4, 16), bits=10),
    "yvyu numpy": lambda: fb.YUV422Frame.yvyu(np.zeros((4, 16), np.uint8)),
    "nv16 odd rows": lambda: fb.YUV422Frame.nv16(_u8(7, 8)),
    "nv16 odd W": lambda: fb.YUV422Frame.nv16(_u8(8, 7)),
    "p210 int16": lambda: fb.YUV422Frame.nv16(torch.zeros(8, 8, dtype=torch.int16), bits=10),
    "i422 not contiguous": lambda: fb.YUV422Frame.i422(_u8(8, 16)[:, ::2]),
    "i422 odd rows": lambda: fb.YUV422Frame.i422(_u8(9, 8)),
    "444 chroma halved": lambda: fb.YUV444Frame(_u8(4, 6), _u8(2, 3), _u8(2, 3)),
    "444 H = 0": lambda: fb.YUV444Frame(_u8(0, 6), _u8(0, 6), _u8(0, 6)),
    "444 mixed dtypes": lambda: fb.YUV444Frame(_u16(4, 6), _u8(4, 6), _u8(4, 6), bits=10),
    "444 luma 3-D": lambda: fb.YUV444Frame(_u8(4, 6, 1), _u8(4, 6), _u8(4, 6)),
    "i444 rows not 3H": lambda: fb.YUV444Frame.i444(_u8(8, 6)),
    "i444 msb at 8 bits": lambda: fb.YUV444Frame.i444(_u8(9, 6), msb=True),
    "i444 bits 9": lambda: fb.YUV444Frame.i444(_u16(9, 6), bits=9),
    "i444 bits True": lambda: fb.YUV444Frame.i444(_u8(9, 6), bits=True),
    "yuyv unknown matrix": lambda: fb.YUV422Frame.yuyv(_u8(4, 16), matrix="bt470"),
    "nv16 bits 16": lambda: fb.YUV422Frame.nv16(_u16(8, 8), bits=16),
    "CPU yuyv": lambda: fb.YUV422Frame.yuyv(_u8(4, 16)),
    "CPU i444": lambda: fb.YUV444Frame.i444(_u8(9, 6)),
    "CPU 420 and 422": lambda: [fb.YUV420Frame.nv12(_u8(6, 8)), fb.YUV422Frame.nv16(_u8(8, 8))],
    "YUYV then RGB": lambda: [fb.YUV422Frame.yuyv(_u8(4, 16)), RGB],
    "RGB then I444": lambda: [RGB, fb.YUV444Frame.i444(_u8(9, 6))],
    "tensor then NV16": lambda: [torch.zeros(4, 8, 3, dtype=torch.uint8), fb.YUV422Frame.nv16(_u8(8, 8))],
    "I444 then tensor": lambda: [fb.YUV444Frame.i444(_u8(9, 6)), torch.zeros(4, 8, 3, dtype=torch.uint8)],
}


@pytest.mark.parametrize("what", list(BAD_FRAMES))
def test_bad_frames_are_refused_before_device_calls(what):
    """Malformed planes, shapes, dtypes, odd sizes and formats are refused by the constructors; well-formed frames in
    host memory, or mixed with RGB frames, by the tracker.  Either way add and update raise ValueError before any
    device call (there is no device here)."""
    make = BAD_FRAMES[what]
    trk = _tracker()
    with pytest.raises(ValueError):
        trk.add(make(), [[1, 1, 2, 2]])
    trk._ids, trk._streams = np.array([0]), np.array([0])
    with pytest.raises(ValueError):
        trk.update(make())


def test_odd_sizes_are_legal_where_chroma_is_not_subsampled():
    assert fb.YUV422Frame(_u8(3, 8), _u8(3, 4), _u8(3, 4)).shape == (3, 8, 3)
    assert fb.YUV422Frame.yuyv(_u8(1, 4)).shape == (1, 2, 3)
    assert fb.YUV444Frame(_u8(3, 5), _u8(3, 5), _u8(3, 5)).shape == (3, 5, 3)
    assert fb.YUV444Frame.i444(_u8(3, 1)).shape == (1, 1, 3)


# ---------------------------------------------------------------------------------------------------- the oracle
def test_oracle_refuses_unknown_subsamplings_and_mismatched_planes():
    y, c = np.zeros((2, 4), np.uint8), np.zeros((2, 2), np.uint8)
    for shift in ((0, 1), (2, 1), (1, 2), (-1, 0)):
        with pytest.raises(ValueError):
            image_ops.yuv_to_rgb(y, c, c, chroma_shift=shift)
    with pytest.raises(ValueError):
        image_ops.yuv_to_rgb(y, c, c, chroma_shift=(0, 0))
    with pytest.raises(ValueError):
        image_ops.yuv_to_rgb(y, c[:1], c[:1], chroma_shift=(1, 0))


def _422_triple_frames():
    """128 frames of 256 x 512 that hold every 8-bit (Y, U, V) triple at 4:2:2: chroma sample (i, j) is (U, V) =
    (i, j), and the two luma samples that share it in frame k are 2k and 2k + 1."""
    u, v = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    for k in range(128):
        y = np.empty((256, 512), np.uint8)
        y[:, 0::2], y[:, 1::2] = 2 * k, 2 * k + 1
        yield y, u, v


def test_422_oracle_is_cv2_yuy2_uyvy_yvyu_on_every_triple():
    """cv2's packed 4:2:2 conversions use the fixed point of its NV12 / I420 conversion, so the default format is
    cv2's bit for bit; the frames are laid out by YUV422Frame's constructors, so the planes they pick out are those
    cv2 reads."""
    for y, u, v in _422_triple_frames():
        want = oracle(y, u, v, (1, 0))
        for layout, code in CV2_PACKED.items():
            (yo, ys), (uo, us), (vo, vs) = PACKED[layout]
            row = np.empty((256, 1024), np.uint8)
            row[:, yo::ys], row[:, uo::us], row[:, vo::vs] = y, u, v
            assert np.array_equal(cv2.cvtColor(row.reshape(256, 512, 2), code), want), layout
            f = getattr(fb.YUV422Frame, layout)(torch.from_numpy(row))
            assert np.array_equal(oracle(f.y.numpy(), f.u.numpy(), f.v.numpy(), (1, 0)), want), layout


def _codes(rng, bits, shape):
    return rng.integers(0, 1 << bits, shape)


@pytest.mark.parametrize("fmt", FORMATS, ids=str)
def test_oracle_at_shifts_1_1_is_yuv420_to_rgb(fmt):
    """Raw samples of every value (noise in whatever bits the reader masks), at every alignment of the bit depth."""
    matrix, full, bits = fmt
    rng = np.random.default_rng(bits)
    dtype = np.uint16 if bits > 8 else np.uint8
    for shift in sorted({0, 16 - bits}) if bits > 8 else (0,):
        y, u, v = (rng.integers(0, np.iinfo(dtype).max + 1, s).astype(dtype) for s in ((64, 90), (32, 45), (32, 45)))
        assert np.array_equal(image_ops.yuv_to_rgb(y, u, v, matrix, full, bits, shift, (1, 1)),
                              image_ops.yuv420_to_rgb(y, u, v, matrix, full, bits, shift))


@pytest.mark.parametrize("fmt", FORMATS, ids=str)
def test_repeated_chroma_at_422_and_444_converts_as_420(fmt):
    """A 4:2:2 frame whose chroma rows are duplicated 4:2:0 rows, and a 4:4:4 frame whose chroma is the nearest
    upsampled 4:2:0 chroma, give yuv420_to_rgb of the 4:2:0 frame; so do the frames the 4:2:2 / 4:4:4 constructors
    read."""
    matrix, full, bits = fmt
    rng = np.random.default_rng(7 + bits)
    y, u, v = _codes(rng, bits, (64, 90)), _codes(rng, bits, (32, 45)), _codes(rng, bits, (32, 45))
    want = oracle(y, u, v, (1, 1), matrix, full, bits)
    u2, v2 = u.repeat(2, 0), v.repeat(2, 0)
    u4, v4 = u2.repeat(2, 1), v2.repeat(2, 1)
    assert np.array_equal(oracle(y, u2, v2, (1, 0), matrix, full, bits), want)
    assert np.array_equal(oracle(y, u4, v4, (0, 0), matrix, full, bits), want)
    fmt_kw = dict(matrix=matrix, full_range=full)
    for layout, (uu, vv), shift in itertools.chain(((lay, (u2, v2), (1, 0)) for lay in ("yuyv_pitched", "nv16", "i422")),
                                                   ((lay, (u4, v4), (0, 0)) for lay in ("i444_pitched", "roi444"))):
        f = ycbcr_frame(y, uu, vv, layout, bits, device="cpu", rng=rng, **fmt_kw)
        got = image_ops.yuv_to_rgb(f.y.numpy(), f.u.numpy(), f.v.numpy(), matrix, full, bits, f.shift, shift)
        assert np.array_equal(got, want), layout
