"""CPU: the HDR specification (image_ops.yuv_to_rgb with ``transfer``, image_ops.hdr_to_sdr and its pieces), the
FearFrameYCbCrHDR record, the frames' hdr_record() and their refusals, and the new C ABI symbols.

The pieces of the chain are checked against equations written here independently (the PQ inverse EOTF, BT.2087's
matrix, BT.2100's HLG reference values), not against the code under test."""
import os
import re

import numpy as np
import pytest
import torch

import feartracker_b200 as fb
from feartracker_b200 import _lib, image_ops
from tests.test_yuv_frames_cpu import RGB, _tracker

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
NEW_SYMBOLS = ("fear_crop_targets_ycbcr_hdr_u8", "fear_advance_targets_ycbcr_hdr", "fear_frame_sums_ycbcr_hdr_u8")
SHIFTS = {"420": (1, 1), "422": (1, 0), "444": (0, 0)}


def _sdr_reference(Y, U, V, matrix, full_range, bits):
    """The H.273 inverse as yuv_to_rgb computed it before transfers existed (codes already masked and upsampled)."""
    _, kr, kb = image_ops.YUV_MATRICES[matrix]
    m = float(1 << (bits - 8))
    if full_range:
        y0, ys, c0 = 0.0, 1.0 / float((1 << bits) - 1), float(1 << (bits - 1))
        cs = ys
    else:
        y0, ys, c0, cs = 16.0 * m, 1.0 / (219.0 * m), 128.0 * m, 1.0 / (224.0 * m)
    kg = (1.0 - kr) - kb
    cr, cb = 2.0 * (1.0 - kr), 2.0 * (1.0 - kb)
    gb, gr = 2.0 * kb * (1.0 - kb) / kg, 2.0 * kr * (1.0 - kr) / kg
    yn = (Y.astype(np.float64) - y0) * ys
    pb = (U.astype(np.float64) - c0) * cs
    pr = (V.astype(np.float64) - c0) * cs
    rgb = [yn + cr * pr, (yn - gb * pb) - gr * pr, yn + cb * pb]
    return np.stack([np.clip(np.rint(255.0 * c), 0, 255) for c in rgb], -1).astype(np.uint8)


@pytest.mark.parametrize("sub", list(SHIFTS))
@pytest.mark.parametrize("bits", [8, 10, 12])
def test_transfer_none_is_the_matrix_alone(sub, bits):
    rng = np.random.default_rng(bits * 7 + len(sub))
    sx, sy = SHIFTS[sub]
    h, w = 6, 10
    dtype = np.uint8 if bits == 8 else np.uint16
    for shift in ((0,) if bits == 8 else (0, 16 - bits)):
        y = (rng.integers(0, 1 << bits, (h, w)) << shift).astype(dtype)
        u, v = ((rng.integers(0, 1 << bits, (h >> sy, w >> sx)) << shift).astype(dtype) for _ in range(2))
        for matrix in image_ops.YUV_MATRICES:
            for full in (False, True):
                a = image_ops.yuv_to_rgb(y, u, v, matrix, full, bits, shift, (sx, sy))
                b = image_ops.yuv_to_rgb(y, u, v, matrix, full, bits, shift, (sx, sy), transfer=None)
                assert np.array_equal(a, b)
                if (matrix, full, bits) != ("bt601", False, 8):
                    mask = (1 << bits) - 1
                    Y = (y.astype(np.int64) >> shift) & mask
                    U, V = (((c.astype(np.int64) >> shift) & mask).repeat(1 << sy, 0).repeat(1 << sx, 1)
                            for c in (u, v))
                    assert np.array_equal(a, _sdr_reference(Y, U, V, matrix, full, bits)), (matrix, full, bits)
                if sub == "420":
                    assert np.array_equal(a, image_ops.yuv420_to_rgb(y, u, v, matrix, full, bits, shift, None))


def _pq_inverse_eotf(fd):
    """SMPTE ST 2084's inverse EOTF, cd/m² -> E', written out from the standard."""
    m1, m2 = 2610 / 16384, 2523 / 4096 * 128
    c1, c2, c3 = 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32
    y = (np.asarray(fd, dtype=np.float64) / 10000.0) ** m1
    return ((c1 + c2 * y) / (1 + c3 * y)) ** m2


def test_pq_eotf_round_trips_through_its_inverse():
    for fd in (0.1, 100.0, 1000.0, 10000.0):
        back = float(image_ops.pq_eotf(_pq_inverse_eotf(fd)))
        assert abs(back - fd) <= 1e-9 * fd, (fd, back)
    assert float(image_ops.pq_eotf(0.0)) == 0.0 and abs(float(image_ops.pq_eotf(1.0)) - 10000.0) < 1e-9


def test_hlg_inverse_oetf_is_continuous_and_gives_bt2100_reference_light():
    lo, hi = np.nextafter(0.5, 0.0), np.nextafter(0.5, 1.0)
    a, b = image_ops.hlg_inverse_oetf(np.array([lo, 0.5, hi]))[[0, 2]]
    assert abs(a - 1 / 12) < 1e-12 and abs(b - 1 / 12) < 1e-12
    assert abs(float(image_ops.hlg_inverse_oetf(1.0)) - 1.0) < 1e-7
    # BT.2408: HLG reference white (75 %) is 203 cd/m² on a 1000 cd/m² display
    light = image_ops.hlg_display_light([np.array(0.75)] * 3)
    assert all(abs(float(c) - 203.0) <= 0.5 for c in light)


def test_method_a_curve_is_continuous_at_its_knots_and_maps_1_to_1():
    """Continuous to the precision of BT.2446-1's 4-digit coefficients: the pieces meet within 5.5e-4 at 0.7399 and
    1.1e-5 at 0.9909, and the curve is monotone across both knots."""
    for knot, gap in ((0.7399, 6e-4), (0.9909, 2e-5)):
        lo, hi = image_ops.method_a_curve(np.array([np.nextafter(knot, 0.0), np.nextafter(knot, 1.0)]))
        assert 0 <= hi - lo < gap, (knot, lo, hi)
    assert (np.diff(image_ops.method_a_curve(np.linspace(0.0, 1.0, 100001))) > 0).all()
    assert float(image_ops.method_a_curve(1.0)) == 1.0


def test_gamut_matrix_rows_sum_to_one_and_match_bt2087():
    m = image_ops.bt2020_to_bt709_matrix()
    assert m.dtype == np.float64 and m.shape == (3, 3)
    assert np.all(np.abs(m.sum(axis=1) - 1.0) < 1e-12)
    bt2087 = np.array([[1.6605, -0.5876, -0.0728], [-0.1246, 1.1329, -0.0083], [-0.0182, -0.1006, 1.1187]])
    assert np.array_equal(np.round(m, 4), bt2087)


def _kernel_source() -> str:
    with open(os.path.join(ROOT, "feartracker_b200", "csrc", "kernels_track_loop.cuh")) as f:
        return f.read()


def test_folded_constants_are_the_kernels_and_their_derivations():
    """Each kHdr* literal of the crop kernel is the hex float of image_ops.HDR_CONSTANTS, and each constant is its
    derivation (within 1 ulp, the most another platform's log or pow may differ by); the gamut matrix literals are
    bt2020_to_bt709_matrix() bit for bit."""
    src = _kernel_source()
    names = {"pq_inv_m1": "kHdrPqInvM1", "pq_inv_m2": "kHdrPqInvM2", "hlg_b": "kHdrHlgB", "hlg_c": "kHdrHlgC",
             "inv_2_4": "kHdrInv24", "rho_hdr_m1": "kHdrRhoHdrM1", "ln_rho_hdr": "kHdrLnRhoHdr",
             "rho_sdr": "kHdrRhoSdr", "rho_sdr_m1": "kHdrRhoSdrM1"}
    assert set(names) == set(image_ops.HDR_CONSTANTS) == set(image_ops.HDR_CONSTANT_DERIVATIONS)
    for key, cname in names.items():
        m = re.search(rf"constexpr double {cname} = (-?0x[0-9a-f.]+p[-+]\d+);", src)
        assert m, cname
        value = image_ops.HDR_CONSTANTS[key]
        assert float.fromhex(m.group(1)) == value, (key, m.group(1), value.hex())
        derived = image_ops.HDR_CONSTANT_DERIVATIONS[key]()
        assert abs(derived - value) <= np.spacing(value), (key, derived, value)
    body = src[src.index("kHdrGamut[3][3] = {"):]
    body = body[:body.index("};")]
    lits = [float.fromhex(t) for t in re.findall(r"-?0x[0-9a-f.]+p[-+]\d+", body)]
    assert lits == image_ops.bt2020_to_bt709_matrix().ravel().tolist()
    assert "kHdrHlgA = 0.17883277;" in src and image_ops.HLG_A == 0.17883277


def _grey(transfer, codes, bits, full):
    """The 8-bit output of neutral pixels (Cb = Cr = mid code) of luma ``codes``, 4:4:4."""
    y = np.asarray(codes, dtype=np.uint16)[None]
    c = np.full_like(y, 1 << (bits - 1))
    return image_ops.yuv_to_rgb(y, c, c, "bt2020", full, bits, 0, (0, 0), transfer)[0]


@pytest.mark.parametrize("transfer", ["pq", "hlg"])
@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("full", [False, True], ids=["limited", "full"])
def test_neutral_inputs_stay_neutral_and_grey_is_monotone(transfer, bits, full):
    out = _grey(transfer, np.arange(1 << bits), bits, full)
    assert (out[:, 0] == out[:, 1]).all() and (out[:, 1] == out[:, 2]).all()
    assert (np.diff(out[:, 0].astype(int)) >= 0).all()
    assert out[0, 0] == 0 and out[-1, 0] == 255


def test_anchors():
    """PQ 100 cd/m² is E' = 0.5081 and maps to 137; HLG E' = 0.75 maps to 175; 1000 cd/m² of either maps to 255."""
    e100 = float(_pq_inverse_eotf(100.0))
    assert abs(e100 - 0.5081) < 5e-5
    for transfer, e, want in (("pq", e100, 137), ("hlg", 0.75, 175), ("pq", float(_pq_inverse_eotf(1000.0)), 255),
                              ("hlg", 1.0, 255)):
        got = image_ops.hdr_to_sdr([np.array([e])] * 3, transfer)
        assert got.tolist() == [[want] * 3], (transfer, e, got)


def test_saturated_colours_stay_in_range_and_keep_their_hue():
    """Pure BT.2020 primaries at HLG reference level come out saturated in the same primary."""
    for i in range(3):
        e = [np.array([0.0])] * 3
        e[i] = np.array([0.75])
        for transfer in ("pq", "hlg"):
            out = image_ops.hdr_to_sdr(e, transfer)[0]
            assert out[i] == out.max() and out[i] > 0, (i, transfer, out)


@pytest.mark.parametrize("args", [dict(transfer="sdr"), dict(transfer=16), dict(transfer="pq", matrix="bt709"),
                                  dict(transfer="hlg", matrix="bt601"), dict(transfer="pq", bits=8)], ids=str)
def test_yuv_to_rgb_refuses_bad_transfers(args):
    kw = dict(matrix="bt2020", bits=10)
    kw.update(args)
    z = np.zeros((2, 2), np.uint16 if kw["bits"] > 8 else np.uint8)
    with pytest.raises(ValueError):
        image_ops.yuv_to_rgb(z, z[:1, :1], z[:1, :1], kw["matrix"], False, kw["bits"], 0, (1, 1), kw["transfer"])


# ---------------------------------------------------------------------------------------------------- record, ABI
def test_hdr_record_is_104_bytes_with_the_header_layout():
    dt = _lib.YCBCR_HDR_DTYPE
    assert dt.itemsize == 104
    assert dt.names == _lib.YCBCR_V210_DTYPE.names + ("transfer", "reserved_hdr")
    assert dt.fields["v210"][1] == 88 and dt.fields["transfer"][1] == 96 and dt.fields["reserved_hdr"][1] == 100
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    body = header[header.index("typedef struct FearFrameYCbCrHDR {"):]
    body = body[:body.index("} FearFrameYCbCrHDR;")]
    fields = []
    for line in body.splitlines()[1:]:
        decl = line.split("/*")[0].strip().rstrip(";")
        if decl:
            fields += [n.strip().lstrip("*") for n in decl.split(None, 2)[-1].split(",")] if decl.startswith("const") \
                else [n.strip() for n in decl.split(None, 1)[1].split(",")]
    assert tuple(fields) == dt.names
    assert "#define FEAR_TRC_PQ 16" in header and "#define FEAR_TRC_HLG 18" in header


def test_new_symbols_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        header = f.read()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header
        assert name in _lib.exported_symbols()
        assert getattr(_lib.load(), name).argtypes
    assert "#define FEAR_ABI_VERSION 1" in header


def _constructors(transfer, bits=10, matrix="bt2020"):
    """Every planar constructor on host tensors (they do not look at the device), at ``bits``."""
    dt = torch.uint8 if bits == 8 else torch.uint16
    kw = dict(matrix=matrix, bits=bits, transfer=transfer)
    y, c = torch.zeros(8, 12, dtype=dt), torch.zeros(4, 6, dtype=dt)
    return {
        "nv12": lambda: fb.YUV420Frame.nv12(torch.zeros(12, 12, dtype=dt), **kw),
        "i420": lambda: fb.YUV420Frame.i420(torch.zeros(12, 12, dtype=dt), **kw),
        "planes420": lambda: fb.YUV420Frame(y, c, c, **kw),
        "yuyv": lambda: fb.YUV422Frame.yuyv(torch.zeros(8, 24, dtype=dt), **kw),
        "uyvy": lambda: fb.YUV422Frame.uyvy(torch.zeros(8, 24, dtype=dt), **kw),
        "yvyu": lambda: fb.YUV422Frame.yvyu(torch.zeros(8, 24, dtype=dt), **kw),
        "nv16": lambda: fb.YUV422Frame.nv16(torch.zeros(16, 12, dtype=dt), **kw),
        "i422": lambda: fb.YUV422Frame.i422(torch.zeros(16, 12, dtype=dt), **kw),
        "i444": lambda: fb.YUV444Frame.i444(torch.zeros(24, 12, dtype=dt), **kw),
    }


@pytest.mark.parametrize("transfer", [None, "pq", "hlg"])
def test_every_constructor_writes_its_hdr_record(transfer):
    code = {None: 0, "pq": 16, "hlg": 18}[transfer]
    for name, make in _constructors(transfer).items():
        f = make()
        assert f.transfer == transfer, name
        rec = f.hdr_record()
        assert rec == f.ycbcr_v210_record() + (code, 0), name
        row = np.array([rec], dtype=_lib.YCBCR_HDR_DTYPE)[0]
        assert (row["transfer"], row["v210"], row["matrix"], row["bits"]) == (code, 0, 2, 10), name
    sdr = fb.YUV420Frame.nv12(torch.zeros(12, 12, dtype=torch.uint8))
    assert sdr.transfer is None and sdr.hdr_record()[-2:] == (0, 0)


BAD = [("unknown name", dict(transfer="hdr10")), ("H.273 code", dict(transfer=16)),
       ("pq with bt709", dict(transfer="pq", matrix="bt709")), ("hlg with bt601", dict(transfer="hlg", matrix="bt601")),
       ("pq at 8 bits", dict(transfer="pq", bits=8)), ("hlg at 8 bits", dict(transfer="hlg", bits=8))]


@pytest.mark.parametrize("what,kw", BAD, ids=[b[0] for b in BAD])
def test_bad_transfers_are_refused_before_device_calls(what, kw):
    """Every constructor raises ValueError for an unknown transfer, an HDR transfer with another matrix than BT.2020 or
    at 8 bits; V210Frame checks the transfer before it looks at its tensor.  So add and update never reach the
    device (there is none here)."""
    kw = dict(dict(matrix="bt2020", bits=10), **kw)
    for name, make in _constructors(kw["transfer"], kw["bits"], kw["matrix"]).items():
        with pytest.raises(ValueError, match="transfer"):
            make()
    if kw["bits"] == 10:
        with pytest.raises(ValueError, match="transfer"):
            fb.V210Frame(torch.zeros(4, 128, dtype=torch.uint8), 48, matrix=kw["matrix"], transfer=kw["transfer"])
    trk = _tracker()
    make = _constructors(kw["transfer"], kw["bits"], kw["matrix"])["nv12"]
    with pytest.raises(ValueError):
        trk.add([make(), RGB], [[1, 1, 2, 2]])
    assert len(trk) == 0


def test_only_calls_with_a_transfer_take_the_hdr_table():
    """ENTRY_POINTS and TABLE_DTYPES name the new table; frames without a transfer keep every existing table."""
    from feartracker_b200 import multi_tracker as multi
    assert multi.ENTRY_POINTS["ycbcr_hdr"] == NEW_SYMBOLS[2:] + NEW_SYMBOLS[:2]
    assert multi.TABLE_DTYPES["ycbcr_hdr"] is _lib.YCBCR_HDR_DTYPE
    from feartracker_b200 import tracker
    assert tracker._TARGET_OFFSET >= _lib.YCBCR_HDR_DTYPE.itemsize and tracker._SMOOTH_OFFSET % 8 == 0
