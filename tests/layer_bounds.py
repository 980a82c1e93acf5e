"""Element-wise fp64 error model of every stage of the hot path, for kernels run in isolation on their own GPU input.

A stage takes a tensor the library exposes (``fear_debug_backbone_prefix``, ``fear_debug_head_tensor``, the maps),
runs the next exposed step of the network on it in float64 from the folded weights the library was packed with, and
compares the result with the library's output element by element.  Every output element i carries three fp64 numbers:

  y_i  the exact result of the stage on the stage's fp32 input;
  E_i  a worst-case bound on |y^_i - y_i| for a correct kernel;
  V_i  a bound on E[(y^_i - y_i)^2] when the rounding errors are modelled as independent random variables.

Two checks follow: (a) |y^ - y| <= E everywhere, which no correct kernel fails and which catches any local error
whatever the element's magnitude; (b) RMS over the stage of |y^ - y| / sqrt(V) <= 1, which catches a precision
regression spread over a whole layer that (a) is far too loose to see.

u = 2^-24 (unit roundoff of fp32).  For a layer output y = sum_k w_k x_k + b (+ r) the magnitude is
S = sum_k |w_k| |x_k| + |b| (+ |r|) and Q^2 = sum_k (w_k x_k)^2.  What each arithmetic contributes:

3xTF32 wgmma GEMM (every 1x1 conv on the tensor cores, csrc/kernels_tc.cuh; K input channels, n = ceil(K/8) steps):
  * load_a_frags: x_hi = x with its 13 low mantissa bits cleared, x_lo = x - x_hi (exact, same sign as x,
    |x_lo| < 2^-10 |x|); the tensor core reads x_lo as tf32, i.e. truncates it: error in (-2^-21 |x|, 0] toward zero,
    <= 8u |x|, mean magnitude <= 4u |x|.
  * fear_pack_weights: w_hi = rna_tf32(w), |w - w_hi| <= 2^-11 |w|; w_lo = rna_tf32(w - w_hi): error <= 2^-22 |w| = 4u |w|,
    unbiased.
  * the x_lo * w_lo term is dropped: |x_lo w_lo| <= 2^-21 |x w| = 8u |x w|, mean magnitude <= 2^-11 * 2^-11 = 4u |x w|.
  * products are exact; each k = 8 step is added to the fp32 accumulator with one rounding, ASSUMED to be a truncation
    of the exact sum of the accumulator and the step's 8 products: error toward zero, < 2^-23 |p_j| = 2u |p_j| for the
    partial sum p_j after step j (|p_j| <= S).  The two correction products of a step go to a second accumulator of
    magnitude < 2^-9 S: < 2^-7 u S per step.
  * epilogue: main + corr, bias + residual, + that sum: three round-to-nearest adds, <= 2u S each counted as a step.
  Worst case: E = (C_REP_GEMM + 2 (n + 4)) u S with C_REP_GEMM = 8 + 4 + 8 + 1 = 21.  This holds for every correct
  kernel only as far as the accumulation assumption holds; how Hopper's wgmma aligns and rounds the 8 products of a
  step inside the tensor core is not documented, and a unit that truncates each product to the largest exponent before
  adding could exceed 2u |p_j| per step.
  Model second moment: truncation errors are not zero-mean, so the bound is the sum of the errors' second moments plus
  the square of the sum of their mean magnitudes (the coherent part, reached when the errors keep their sign, e.g. with
  non-negative operands).  A truncation error in [0, 2u|p|) has second moment <= (4/3) u^2 p^2 and mean <= u |p|; a
  round-to-nearest error is zero-mean with second moment <= u^2 S^2 / 3; the representation errors have second moments
  (8^2 + 4^2 + 8^2) / 3 = 48 u^2 (w x)^2 per product and mean magnitudes 4u + 4u = 8u |w x|.  With P = sum_k |w_k x_k|
  and the exact partial sums p_j of the kernel's K order:
      V = u^2 ((4/3) sum_j p_j^2 + S^2 + 48 Q^2 + (sum_j |p_j| + 2^-7 n S + 8 P)^2).

3xTF32 correlation (corr_tc_kernel, K = 256, n = 32): both operands are split by truncation in the kernel (z_lo is
  written to shared memory exact and truncated by the tensor core, like x_lo): 8u + 8u, and the dropped lo * lo term is
  < 2^-20 = 16u.  C_REP_CORR = 8 + 8 + 16 + 1 = 33; representation second moments (8^2 + 8^2 + 16^2) / 3 = 128 u^2 (z x)^2
  and mean magnitudes 4u + 4u + 4u = 12u |z x|; the accumulation terms are those of the GEMM.

CUDA-core FFMA (depthwise 3x3 / 5x5, the stem, pw=ffma, corr=ffma, fear_corr_concat_f32, the 16x16 / 24x24 1x1
  convs, the prediction convs): every fma / add rounds to nearest, error <= u |partial| <= u S.  K products, the bias
  and a residual: E = (K + 2) u S, V = (K + 2) u^2 S^2 / 3.  The prediction conv (pred_pw_kernel) sums 8 products per
  lane and a 5-level shuffle tree, then the bias: 14 roundings, E = 15 u S.

bbox = exp(z) (expf, <= 2 ulp): compared as log(bbox^) - z, whose error is that of z plus <= 2 * 2u.

Stages with unexposed intermediates (a backbone block: pw -> dw -> pwl (+x); a SepConv: dw -> pw; a tower: two
SepConvs) carry the error bounds through: E_out = |W| * E_in + E_own and V_out = W^2 * V_in + V_own (ReLU is
1-Lipschitz and passes both on).  The magnitude used for a layer's own rounding is that of its exact input.
"""
import math
from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.fbnet_c import FBNET_C, NUM_HOT_BLOCKS

U = 2.0 ** -24
C_REP_GEMM, VAR_REP_GEMM, MEAN_REP_GEMM = 21, 48.0, 8.0
C_REP_CORR, VAR_REP_CORR, MEAN_REP_CORR = 33, 128.0, 12.0
EXP_ULPS = 2
PRED_ROUNDINGS = 14

# The 16 blocks the library runs (FBNET_C without the stem and the skip block), in the order of
# fear_debug_backbone_prefix's nblocks.
BLOCKS = [s for s in FBNET_C[1:NUM_HOT_BLOCKS] if s.kind == "ir"]


class Est(NamedTuple):
    """An activation with its per-element error model (all float64, NCHW)."""
    y: torch.Tensor
    E: torch.Tensor  # worst-case absolute error bound
    V: torch.Tensor  # model second moment of the error


def exact(x: torch.Tensor) -> Est:
    """An fp32 tensor the library exposed: taken as exact input of the next stage."""
    y = x.detach().to("cpu", torch.float64)
    z = torch.zeros_like(y)
    return Est(y, z, z.clone())


# ------------------------------------------------------------------------------------------------ layer arithmetic
class Model(NamedTuple):
    """Own rounding of one layer: E += a u S; V += u^2 (vs S^2 + vq Q^2 + ((4/3) sum p_j^2 + (sum |p_j| + 2^-7 n S +
    m P)^2 when n > 0)), where n is the number of truncating k = 8 tensor-core steps (0: round-to-nearest only)."""
    a: float
    vs: float
    vq: float
    m: float = 0.0
    n: int = 0


def gemm_model(K: int) -> Model:
    """3xTF32 1x1 conv over K input channels."""
    n = -(-K // 8)
    return Model(C_REP_GEMM + 2 * (n + 4), 1.0, VAR_REP_GEMM, MEAN_REP_GEMM, n)


def corr_model() -> Model:
    """3xTF32 pixel-wise correlation (K = 256); its epilogue is the one main + corr add."""
    return Model(C_REP_CORR + 2 * (32 + 4), 1.0 / 3.0, VAR_REP_CORR, MEAN_REP_CORR, 32)


def ffma_model(n_round: int) -> Model:
    """Round-to-nearest CUDA-core arithmetic with n_round roundings, each <= u S."""
    return Model(float(n_round), n_round / 3.0, 0.0)


def _steps(chunks: torch.Tensor):
    """chunks [..., n, ...] (dim 2 = the k = 8 steps in K order) -> (sum_j |p_j|, sum_j p_j^2) of the partial sums."""
    p = chunks.cumsum(2)
    return p.abs().sum(2), (p * p).sum(2)


def _own(model: Model, S, Q2, P, steps=None):
    """(E, V) of a layer's own rounding (see Model)."""
    E = model.a * U * S
    V = model.vs * S * S + model.vq * Q2
    if model.n:
        A, P2 = steps
        V = V + (4.0 / 3.0) * P2 + (A + 2.0 ** -7 * model.n * S + model.m * P) ** 2
    return E, U * U * V


def conv(x: Est, w: torch.Tensor, b: Optional[torch.Tensor], model: Model, stride: int = 1, groups: int = 1,
         relu: bool = False, res: Optional[Est] = None) -> Est:
    """One conv layer (kxk, padding k//2) of the stage with its own rounding model (see module docstring).  Tensor-core
    models (model.n > 0) are 1x1 convs."""
    pad = w.shape[-1] // 2
    aw = w.abs()
    y = F.conv2d(x.y, w, b, stride, pad, 1, groups)
    P = F.conv2d(x.y.abs(), aw, None, stride, pad, 1, groups)
    Q2 = F.conv2d(x.y * x.y, w * w, None, stride, pad, 1, groups)
    E = F.conv2d(x.E, aw, None, stride, pad, 1, groups)
    V = F.conv2d(x.V, w * w, None, stride, pad, 1, groups)
    S = P if b is None else P + b.abs().view(1, -1, 1, 1)
    if res is not None:
        y, S, E, V = y + res.y, S + res.y.abs(), E + res.E, V + res.V
    steps = None
    if model.n:
        B, K, H, W = x.y.shape
        pad_k = 8 * model.n - K
        xs = F.pad(x.y, (0, 0, 0, 0, 0, pad_k)).view(B, model.n, 8, H, W)
        ws = F.pad(w[:, :, 0, 0], (0, pad_k)).view(w.shape[0], model.n, 8)
        steps = _steps(torch.einsum("bjkhw,njk->bnjhw", xs, ws))
    Eo, Vo = _own(model, S, Q2, P, steps)
    if relu:
        y = torch.relu(y)
    return Est(y, E + Eo, V + Vo)


def pw_model(K: int, cin: int, cout: int, pw: str):
    """Which arithmetic the library uses for a 1x1 conv: the 16x16 / 24x24 layers always run on CUDA cores
    (pw_small_const_kernel, the fused stem and expand-1 kernels), every other one on the tensor cores unless pw=ffma."""
    if pw == "ffma" or (cin, cout) in ((16, 16), (24, 24)):
        return ffma_model(K + 2)
    return gemm_model(K)


# ------------------------------------------------------------------------------------------------ folded weights
def unpack(blob: np.ndarray, offsets: np.ndarray, table) -> Dict[str, torch.Tensor]:
    """The fp32 blob fear_pack_weights consumed -> float64 tensors in torch conv layout, keyed by library name."""
    out = {}
    for i, (name, numel) in enumerate(table):
        a = torch.from_numpy(np.asarray(blob[int(offsets[i]):int(offsets[i + 1])], dtype=np.float64).copy())
        assert a.numel() == numel, name
        out[name] = a
    shaped = {"stem.w": out["stem.w"].view(16, 3, 3, 3), "stem.b": out["stem.b"]}
    for s in BLOCKS:
        if s.expand != 1:
            shaped[s.name + ".pw.w"] = out[s.name + ".pw.w"].view(s.mid, s.cin, 1, 1)
            shaped[s.name + ".pw.b"] = out[s.name + ".pw.b"]
        shaped[s.name + ".dw.w"] = out[s.name + ".dw.w"].view(s.mid, 1, s.k, s.k)
        shaped[s.name + ".dw.b"] = out[s.name + ".dw.b"]
        shaped[s.name + ".pwl.w"] = out[s.name + ".pwl.w"].view(s.cout, s.mid, 1, 1)
        shaped[s.name + ".pwl.b"] = out[s.name + ".pwl.b"]
    shaped["neck.w"], shaped["neck.b"] = out["neck.w"].view(256, 112, 1, 1), out["neck.b"]
    for name in list(out):
        if name in shaped or name.startswith(("stem.", "xif", "neck.")):
            continue
        if name.endswith(".dw.w"):
            shaped[name] = out[name].view(-1, 1, 3, 3)
        elif name.endswith(".pw.w"):
            cout = out[name[:-1] + "b"].numel()
            shaped[name] = out[name].view(cout, -1, 1, 1)
        else:
            shaped[name] = out[name]
    return shaped


# ------------------------------------------------------------------------------------------------ stages
def stem(W, img: Est) -> Est:
    """xif0_0: 3x3 stride 2 conv + bias + ReLU on the normalised image (27 FMAs after the bias)."""
    return conv(img, W["stem.w"], W["stem.b"], ffma_model(27 + 2), stride=2, relu=True)


def block(W, n: int, x: Est, pw: str = "auto") -> Est:
    """Backbone block n (0-based, xif1_0 .. xif4_7): [pw 1x1 + ReLU] -> dw kxk + ReLU -> pwl 1x1 (+ x)."""
    s = BLOCKS[n]
    h = x
    if s.expand != 1:
        h = conv(h, W[s.name + ".pw.w"], W[s.name + ".pw.b"], pw_model(s.cin, s.cin, s.mid, pw), relu=True)
    h = conv(h, W[s.name + ".dw.w"], W[s.name + ".dw.b"], ffma_model(s.k * s.k + 2), stride=s.stride, groups=s.mid,
             relu=True)
    return conv(h, W[s.name + ".pwl.w"], W[s.name + ".pwl.b"], pw_model(s.mid, s.mid, s.cout, pw),
                res=x if s.residual else None)


def neck(W, x: Est, pw: str = "auto") -> Est:
    return conv(x, W["neck.w"], W["neck.b"], pw_model(112, 112, 256, pw))


def sepconv(W, prefix: str, x: Est, pw: str = "auto") -> Est:
    """Head SepConv (folded BN): depthwise 3x3 without bias -> 1x1 + bias + ReLU."""
    c = x.y.shape[1]
    d = conv(x, W[prefix + ".dw.w"], None, ffma_model(9 + 2), groups=c)
    return conv(d, W[prefix + ".pw.w"], W[prefix + ".pw.b"], pw_model(c, c, 256, pw), relu=True)


def correlation(z: Est, x: Est, corr: str = "auto") -> Est:
    """s[b, k, p] = sum_c z[b, c, k] x[b, c, p] (pixel-wise correlation, K = 256): z (Bz, 256, 8, 8) with Bz = 1
    broadcast, x (B, 256, 16, 16) -> (B, 64, 16, 16)."""
    B = x.y.shape[0]
    zy = z.y.reshape(z.y.shape[0], 256, 64).expand(B, 256, 64)
    xy = x.y.reshape(B, 256, 256)
    y = torch.bmm(zy.transpose(1, 2), xy)
    S = torch.bmm(zy.abs().transpose(1, 2), xy.abs())
    Q2 = torch.bmm((zy * zy).transpose(1, 2), xy * xy)
    if corr == "ffma":
        E, V = _own(ffma_model(256 + 2), S, Q2, S)
    else:
        chunks = torch.einsum("bjck,bjcp->bkjp", zy.reshape(B, 32, 8, 64), xy.reshape(B, 32, 8, 256))
        E, V = _own(corr_model(), S, Q2, S, _steps(chunks))
    shape = (B, 64, 16, 16)
    return Est(y.view(shape), E.view(shape), V.view(shape))


def tower(W, name: str, x: Est, pw: str = "auto") -> Est:
    """bbox_tower / cls_tower: two SepConvs, the middle activation never leaves the library."""
    return sepconv(W, name + ".1", sepconv(W, name + ".0", x, pw), pw)


def pred(W, name: str, x: Est) -> Est:
    """bbox_pred / cls_pred: depthwise 3x3 then pred_pw_kernel (bbox: the argument of its exp)."""
    d = conv(x, W[name + ".dw.w"], None, ffma_model(9 + 2), groups=256)
    return conv(d, W[name + ".pw.w"], W[name + ".pw.b"], ffma_model(PRED_ROUNDINGS + 1))


# ------------------------------------------------------------------------------------------------ checks
def compare(got: torch.Tensor, want: Est, log_of_exp: bool = False) -> Dict[str, float]:
    """(a) max |y^ - y| / E and (b) RMS |y^ - y| / sqrt(V) of one stage; both must be <= 1, and "nonfinite" counts the
    output elements that are not finite (after the log) -- there must be none.  With log_of_exp the stage output is
    exp(y) and log(y^) is compared (the exp's own rounding is added to the bounds)."""
    g = got.detach().to("cpu", torch.float64)
    E, V = want.E, want.V
    if log_of_exp:
        g = torch.log(g)
        E = E + 2 * EXP_ULPS * U
        V = V + (2 * EXP_ULPS * U) ** 2 / 3
    err = (g - want.y).abs()
    a = torch.where(E > 0, err / E.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    b = torch.where(V > 0, err * err / V.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    bad = int((~torch.isfinite(g)).sum())
    return {"a": float(a.max()), "b": float(b.mean().sqrt()), "nonfinite": bad}


def legacy_inf_norm(got: torch.Tensor, want: torch.Tensor) -> float:
    """The inf-norm metric of the existing suite (tests/helpers.map_errors (ii))."""
    g = got.detach().to("cpu", torch.float64)
    return float((g - want).abs().max() / want.abs().max().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------ weight sets
def _round_tf32(a: np.ndarray) -> np.ndarray:
    """fp32 -> tf32 round to nearest, ties away (cvt.rna.tf32.f32 / host_rna_tf32), kept in fp32."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def is_gemm_weight(name: str) -> bool:
    """The tensors fear_pack_weights splits into tf32 (hi, lo) pairs."""
    return not name.startswith(("bbox_pred", "cls_pred")) and (
        name.endswith(".pw.w") or name.endswith(".pwl.w") or name == "neck.w")


def synthetic_folded(table, seed: int, wide: bool, tf32_exact: bool) -> Dict[str, np.ndarray]:
    """A seeded folded weight set in library order (float32 per tensor, full random mantissas).

    Every conv has He-scaled normal weights (sqrt(2 / fan_in), sqrt(1 / fan_in) before no ReLU) so activations keep
    their scale over the 40 layers.  wide=True multiplies each output channel's weights and bias of every conv by a
    log-uniform factor in [2^-8, 2^8] (divided by the RMS of the factors, which keeps the layer's gain): every layer then
    has channels ~10^4 below its largest.  tf32_exact=True rounds the GEMM weights to tf32, so w_lo = 0 and the whole
    3xTF32 correction comes from the activation split.  The bbox prediction is scaled so that its exp stays near 1."""
    rng = np.random.default_rng(seed)
    out = {}
    names = [n for n, _ in table]
    numel = dict(table)
    for name in names:
        if not name.endswith(".w"):
            continue
        base = name[:-2]
        n_out = numel[base + ".b"] if base + ".b" in numel else None
        if name.endswith(".dw.w") or name == "stem.w":
            n_out = numel[name] // (27 if name == "stem.w" else (9 if not name.startswith("xif") else
                                    next(s.k * s.k for s in BLOCKS if name == s.name + ".dw.w")))
        fan_in = numel[name] // n_out
        relu = not (name.endswith(".pwl.w") or name == "neck.w" or "pred" in name or
                    (name.endswith(".dw.w") and not name.startswith("xif")))
        w = rng.standard_normal((n_out, fan_in)) * math.sqrt((2.0 if relu else 1.0) / fan_in)
        b = rng.standard_normal(n_out) * 0.1
        if wide:
            s = 2.0 ** rng.uniform(-8, 8, n_out)
            s /= np.sqrt(np.mean(s * s))
            w *= s[:, None]
            b *= s
        if name.startswith("bbox_pred"):
            w *= 0.002
        out[name] = w.reshape(-1).astype(np.float32)
        if base + ".b" in numel:
            out[base + ".b"] = b.astype(np.float32)
    for name in names:
        if tf32_exact and is_gemm_weight(name):
            out[name] = _round_tf32(out[name])
    return {n: out[n] for n in names}


def blob_of(folded: Dict[str, np.ndarray], table) -> Tuple[np.ndarray, np.ndarray]:
    """Folded tensors -> (fp32 blob, uint64 offsets) in the library's fear_weight_name / fear_weight_numel order."""
    offsets = np.zeros(len(table) + 1, dtype=np.uint64)
    chunks = []
    for i, (name, numel) in enumerate(table):
        a = np.ascontiguousarray(folded[name], dtype=np.float32).reshape(-1)
        assert a.size == numel, (name, a.size, numel)
        chunks.append(a)
        offsets[i + 1] = offsets[i] + np.uint64(numel)
    return np.concatenate(chunks), offsets


def weight_sets(state_dict, table) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """The three blobs the tests pack: the checkpoint, a wide-scale set and a set with tf32-exact GEMM weights."""
    from feartracker_b200 import weights

    return {
        "checkpoint": weights.pack(state_dict, table),
        "wide": blob_of(synthetic_folded(table, 101, wide=True, tf32_exact=False), table),
        "tf32_exact": blob_of(synthetic_folded(table, 202, wide=False, tf32_exact=True), table),
    }


# ------------------------------------------------------------------------------------------------ inputs
def normalize_u8(u8_nhwc: np.ndarray) -> torch.Tensor:
    """(B, H, W, 3) uint8 -> (B, 3, H, W) float32 normalised exactly as the tracker (and the stem kernel) does it."""
    from oracle import fear_oracle as fo

    return torch.from_numpy(np.stack([fo.normalize_image(i) for i in u8_nhwc])).permute(0, 3, 1, 2).contiguous()


def input_crops(H: int, W: int) -> Dict[str, np.ndarray]:
    """Named (H, W, 3) uint8 crops: uniform noise, two tracker crops of the demo clip (recorded search crops at
    256 x 256, the template crop at 128 x 128), a constant padding-colour crop (an invalid target's crop) and a 0/255
    checkerboard."""
    import os

    from tests.helpers import GOLDEN

    g = torch.Generator().manual_seed(H * 1000 + W)
    crops = {"noise": torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).numpy()}
    with np.load(os.path.join(GOLDEN, "video_teacher.npz")) as v:
        sc, tc = v["search_crops"], v["template_crop"]
    if (H, W) == (256, 256):
        crops["video_a"], crops["video_b"] = sc[0], sc[4]
    elif (H, W) == (128, 128):
        crops["video_a"] = tc
    else:
        crops["video_a"] = sc[0][64:192]
    pad = np.clip(np.rint(sc[0].reshape(-1, 3).mean(0)), 0, 255).astype(np.uint8)
    crops["constant"] = np.broadcast_to(pad, (H, W, 3)).copy()
    yy, xx = np.mgrid[:H, :W]
    crops["checker"] = np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[:, :, None], 3, axis=2)
    return crops
