"""Tile schedule of the persistent kernels, modelled on the host (plain Python, no CUDA).

Two kernels of the library are persistent: dw_tma_kernel (csrc/kernels_dw_tma.cuh) and dw3_pw24_fused_kernel
(csrc/kernels_dwpw_small.cuh).  Both launch G = min(S, T) CTAs for T tiles on S SMs; CTA c walks the tiles c, c + G,
c + 2G, ... through a 4-stage TMA ring, two consumer groups take alternate tiles, a group refills a stage with the tile
4G ahead, and every barrier wait uses the parity (it / 4) & 1 of the CTA's iteration it.  A fault in that logic only
shows once a CTA gets enough tiles: a wrong parity at its 9th tile (third use of a stage), a wrong refill predicate
when CTAs end on different laps, a group mix-up when a CTA has an odd number of tiles.

`launches()` lists every kernel launch of one chunk of an entry point (get_features, fear_track_u8, fear_head) in the
order fear_context.cu issues them, mirroring the guards of run_backbone / run_blocks / launch_dw / launch_sepconv /
run_head and the tile formulas of launch_dw_tma_t and launch_dw3_pw24.  Its length is the launch count of the call
(tests/schedule_check.py compares it with fear_launch_count, so this model cannot drift silently from the executor).
`plan()` picks, for every persistent launch, the smallest batch that reaches each scheduling regime (REGIMES).
"""
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

STAGES, GROUPS = 4, 2  # TMA ring depth and consumer groups of both persistent kernels
DW_CB = 32             # channels per dw_tma_kernel tile
H100_SXM_SMS, H100_PCIE_SMS = 132, 114

# kBlocks of csrc/arch.h: name, cin, cout, k, stride, expand
BLOCKS = [("xif1_0", 16, 16, 3, 1, 1), ("xif2_0", 16, 24, 3, 2, 6), ("xif2_2", 24, 24, 3, 1, 1),
          ("xif2_3", 24, 24, 3, 1, 1), ("xif3_0", 24, 32, 5, 2, 6), ("xif3_1", 32, 32, 5, 1, 3),
          ("xif3_2", 32, 32, 5, 1, 6), ("xif3_3", 32, 32, 3, 1, 6), ("xif4_0", 32, 64, 5, 2, 6),
          ("xif4_1", 64, 64, 5, 1, 3), ("xif4_2", 64, 64, 5, 1, 6), ("xif4_3", 64, 64, 5, 1, 6),
          ("xif4_4", 64, 112, 5, 1, 6), ("xif4_5", 112, 112, 5, 1, 6), ("xif4_6", 112, 112, 5, 1, 6),
          ("xif4_7", 112, 112, 5, 1, 3)]
FS_TH, FS_TW = 16, 32     # fused stem + xif1_0 output tile (kernels_stem_fused.cuh)
IRF_TH, IRF_TW = 8, 16    # fused xif2_0 output tile (kernels_irf_fused.cuh)
DP_TILE = 16              # dw3_pw24_fused_kernel output tile (16 x 16)
FEAT_C, CAT_C, BACKBONE_C, SCORE, TMPL_PIX = 256, 320, 112, 16, 64
CORR_A_BYTES, PW_MAX_SMEM = 128 * 128, 232448 - 1024  # kernels_tc.cuh

DEFAULTS = {"fuse_stem": "1", "fuse_irf": "1", "fuse_dwpw": "15", "dw": "auto", "pw": "auto", "corr": "auto",
            "pdl": "1"}
DW_CODES = {"pixel": 0, "strip": 1, "roll": 2, "auto": 3, "tma": 6}

# Batch caps per crop size: the sweep of every option set stays short on the GPU.
BATCH_CAPS = {(256, 256): 320, (128, 128): 600, (128, 256): 320}

# (regime, description); a regime is reached by one launch of T = B * t tiles on S SMs, G = min(S, T) CTAs
REGIMES = [
    ("under_one_wave", "T < S: every CTA has one tile"),
    ("first_partial_wave", "S <= T < S + t: the first batch that fills every SM"),
    ("cta_2_tiles", "a CTA with exactly 2 tiles"),
    ("cta_3_tiles", "a CTA with exactly 3 tiles"),
    ("cta_5_tiles", "a CTA with exactly 5 tiles: its first stage refill"),
    ("cta_9plus_tiles", "a CTA with >= 9 tiles: the barrier parity wraps"),
    ("cta_9plus_uneven", ">= 9 tiles with T mod G != 0: CTAs end on different laps"),
    ("busiest_odd", "the busiest CTA has an odd tile count >= 3: its groups end on different tile counts"),
]
REGIME_NAMES = [r for r, _ in REGIMES]


@dataclass(frozen=True)
class Launch:
    """One kernel launch.  Persistent launches carry their tiling: tiles_x * tiles_y pixel tiles of th x tw outputs
    per frame, times cblocks 32-channel blocks (dw_tma_kernel: tile index = ((b * tiles_y + ty) * tiles_x + tx) *
    cblocks + cb; dw3_pw24_fused_kernel: cblocks = 1)."""
    name: str
    kernel: str = "other"
    tiles_x: int = 0
    tiles_y: int = 0
    cblocks: int = 0
    th: int = 0
    tw: int = 0

    @property
    def persistent(self) -> bool:
        return self.kernel != "other"

    @property
    def tiles(self) -> int:
        """Tiles per frame."""
        return self.tiles_x * self.tiles_y * self.cblocks


class _Opt:
    def __init__(self, opts: Optional[Dict[str, str]]):
        o = dict(DEFAULTS)
        o.update(opts or {})
        unknown = set(o) - set(DEFAULTS)
        if unknown:
            raise ValueError(f"unknown options {sorted(unknown)}")
        self.fuse_stem = int(o["fuse_stem"]) != 0
        self.fuse_irf = int(o["fuse_irf"]) != 0
        self.fuse_dwpw = int(o["fuse_dwpw"]) & 15
        self.dw = DW_CODES[o["dw"]]
        self.pw_tc = o["pw"] != "ffma"      # auto = wgmma on an H100
        self.corr_tc = o["corr"] != "ffma"


def _pw_tile_n(n: int) -> int:
    np_ = (n + 15) & ~15
    tiles = (np_ + 127) // 128
    need = (np_ + tiles - 1) // tiles
    return next((nt for nt in (16, 32, 48, 64, 96, 112, 128) if nt >= need), 0)


def _pw_dw_takes(dw_k: int, k: int, n: int, map_w: int) -> bool:
    """tc::launch_pw_dw accepts the shape (else it returns 1 and the caller runs depthwise and 1x1 separately)."""
    if dw_k not in (3, 5) or k % 4 or map_w not in (16, 32):
        return False
    nt = _pw_tile_n(n)
    if not nt:
        return False
    box = (128 // map_w + dw_k - 1) * (map_w + dw_k - 1) * 128
    stage = (CORR_A_BYTES + 2 * nt * 128 + box + dw_k * dw_k * 128 + 128 + 1023) & ~1023
    stages = 1 if (k + 31) // 32 < 2 else 2
    return stages * stage + 1024 + 256 <= PW_MAX_SMEM


def _dw(name, c, k, stride, relu, bias, h, w, opt: _Opt) -> Launch:
    """launch_dw: one launch, a persistent dw_tma_kernel where the TMA pipeline takes the layer."""
    want_tma = opt.dw in (3, 6)
    ho, wo = h // stride, w // stride
    if want_tma and stride == 2 and k == 5 and relu and bias and ho % 8 == 0 and wo % 8 == 0 and c % 4 == 0:
        return Launch(name, "dw_tma<5,2>", wo // 8, ho // 8, math.ceil(c / DW_CB), 8, 8)
    instantiated = (k in (3, 5) and relu and bias) or (k == 3 and not relu and not bias)
    if want_tma and stride == 1 and c >= 24 and instantiated and h % 16 == 0 and w % 16 == 0 and c % 4 == 0:
        kind = f"dw_tma<{k},1>" if bias else f"dw_tma<{k},1,no bias>"
        return Launch(name, kind, w // 16, h // 16, math.ceil(c / DW_CB), 16, 16)
    return Launch(name)


def backbone(H: int, W: int, opt: _Opt, fused_stem_allowed: bool = True) -> List[Launch]:
    """run_backbone (fused_stem_allowed = False: fear_debug_backbone_prefix, which always runs the plain stem)."""
    out = []
    fuse_stem = fused_stem_allowed and opt.fuse_stem and (H // 2) % FS_TH == 0 and (W // 2) % FS_TW == 0
    out.append(Launch("stem+xif1_0" if fuse_stem else "stem"))
    h, w = H // 2, W // 2
    for i, (name, cin, cout, k, stride, e) in enumerate(BLOCKS):
        if i == 0 and fuse_stem:
            continue
        mid, has_pw, residual = cin * e, e != 1, stride == 1 and cin == cout
        if i == 1 and opt.fuse_irf and opt.pw_tc and h % 2 == 0 and w % 2 == 0 and (h // 2) % IRF_TH == 0 \
                and (w // 2) % IRF_TW == 0:
            out.append(Launch(name + " fused"))
            h, w = h // 2, w // 2
            continue
        if (opt.fuse_dwpw & 8) and not has_pw and stride == 1 and k == 3 and cin == 24 and cout == 24 and residual \
                and opt.pw_tc and h % DP_TILE == 0 and w % DP_TILE == 0:
            out.append(Launch(name + " dw+pw", "dw3_pw24", w // DP_TILE, h // DP_TILE, 1, DP_TILE, DP_TILE))
            continue
        if has_pw:
            out.append(Launch(name + ".pw"))
        if (opt.fuse_dwpw & 1) and stride == 1 and has_pw and w == h and (h == 16 or (h == 32 and opt.fuse_dwpw & 4)) \
                and opt.pw_tc and _pw_dw_takes(k, mid, cout, h):
            out.append(Launch(name + ".dw+pwl"))
            continue
        out.append(_dw(name + ".dw", mid, k, stride, True, True, h, w, opt))
        h, w = h // stride, w // stride
        out.append(Launch(name + ".pwl"))
    return out


def head(opt: _Opt) -> List[Launch]:
    """run_head without an update template."""
    out = []

    def sepconv(name, c):
        if (opt.fuse_dwpw & 2) and opt.pw_tc and _pw_dw_takes(3, c, FEAT_C, SCORE):
            out.append(Launch(name + " dw+pw"))
        else:
            out.append(_dw(name + ".dw", c, 3, 1, False, False, SCORE, SCORE, opt))
            out.append(Launch(name + ".pw"))

    for br in ("cls", "reg"):
        sepconv(br + "_encode", FEAT_C)
    out += [Launch("corr")] if opt.corr_tc else [Launch("corr cls"), Launch("corr reg")]
    for br in ("cls", "reg"):
        sepconv(br + "_dw", CAT_C)
    for tower, pred in (("bbox_tower", "bbox_pred"), ("cls_tower", "cls_pred")):
        for i in range(2):
            sepconv(f"{tower}.{i}", FEAT_C)
        out.append(_dw(pred + ".dw", FEAT_C, 3, 1, False, False, SCORE, SCORE, opt))
        out.append(Launch(pred + ".pw"))
    return out


def launches(entry: str, H: int = 256, W: int = 256, opts: Optional[Dict[str, str]] = None, Bz: int = 0,
             boxes: bool = True) -> List[Launch]:
    """Launches of one call whose batch fits the reserved workspace (one chunk).
    entry: "get_features" (float or uint8: the same kernels), "track_u8" (fear_track_u8 at 256 x 256, template
    batch Bz = 1 or B, boxes = whether FearBox records are requested) or "head" (fear_head, template batch Bz)."""
    opt = _Opt(opts)
    if entry == "get_features":
        return backbone(H, W, opt) + [Launch("neck"), Launch("transpose")]
    if entry == "track_u8":
        return ([Launch("stage template")] + backbone(256, 256, opt) + [Launch("neck")] + head(opt)
                + ([Launch("decode")] if boxes else []))
    if entry == "head":
        return [Launch("stage template"), Launch("transpose search")] + head(opt)
    if entry == "backbone_prefix":
        return backbone(H, W, opt, fused_stem_allowed=False)
    raise ValueError(entry)


# --------------------------------------------------------------------------------------------------------- regimes
def cta_tile_counts(T: int, S: int) -> Tuple[int, int]:
    """(G, busiest) for T tiles on S SMs; CTA c has ceil((T - c) / G) tiles, so counts are q or q + 1."""
    G = min(S, T)
    return G, -(-T // G)


def in_regime(regime: str, T: int, S: int, t: int) -> bool:
    G, busiest = cta_tile_counts(T, S)
    q, r = divmod(T, G)
    counts = {q, q + 1} if r else {q}
    if regime == "under_one_wave":
        return T < S
    if regime == "first_partial_wave":
        return S <= T < S + t
    if regime.startswith("cta_") and regime.endswith("_tiles") and regime[4:-6].isdigit():
        return int(regime[4:-6]) in counts
    if regime == "cta_9plus_tiles":
        return busiest >= 9
    if regime == "cta_9plus_uneven":
        return busiest >= 9 and T % G != 0
    if regime == "busiest_odd":
        return busiest >= 3 and busiest % 2 == 1
    raise ValueError(regime)


def smallest_batch(regime: str, t: int, S: int, limit: int = 1 << 16) -> Optional[int]:
    return next((B for B in range(1, limit + 1) if in_regime(regime, B * t, S, t)), None)


def tile_owner(launch: Launch, B: int, S: int, frame: int, y: int, x: int, cb: int = 0) -> Dict[str, int]:
    """Which tile of a persistent launch covers output pixel (y, x) of `frame` in channel block cb, and which CTA,
    iteration, ring stage, barrier parity and consumer group handle it at batch B on S SMs."""
    tile = ((frame * launch.tiles_y + y // launch.th) * launch.tiles_x + x // launch.tw) * launch.cblocks + cb
    G = min(S, B * launch.tiles)
    it = tile // G
    return {"tile": tile, "cta": tile % G, "iteration": it, "stage": it % STAGES, "parity": (it // STAGES) & 1,
            "group": it % GROUPS, "grid": G}


def plan(entry: str, H: int = 256, W: int = 256, opts: Optional[Dict[str, str]] = None, S: int = H100_SXM_SMS,
         **kw) -> Dict[int, List[str]]:
    """Batch -> the "launch: regime" pairs it is the smallest batch for, over every persistent launch of one call.
    Launches with the same tiles per frame share their batches."""
    out: Dict[int, List[str]] = {}
    for ln in launches(entry, H, W, opts, **kw):
        if not ln.persistent:
            continue
        for regime in REGIME_NAMES:
            B = smallest_batch(regime, ln.tiles, S)
            if B is None:
                raise ValueError(f"{ln.name} ({ln.tiles} tiles per frame) never reaches {regime} on {S} SMs")
            out.setdefault(B, []).append(f"{ln.name} [{ln.kernel}, {ln.tiles}/frame]: {regime}")
    return dict(sorted(out.items()))


# Option variants of the GPU sweep.  BIT_IDENTICAL promise the default's arithmetic in the default's order; pw=ffma and
# corr=ffma compute differently, so each frame is compared with the variant's own B = 1 result.
BIT_IDENTICAL = [("fuse_stem", "0"), ("fuse_irf", "0"), ("fuse_dwpw", "0"), ("fuse_dwpw", "14"), ("fuse_dwpw", "11"),
                 ("fuse_dwpw", "13"), ("fuse_dwpw", "7"), ("dw", "pixel"), ("dw", "strip"), ("dw", "roll"),
                 ("dw", "tma"), ("pdl", "0")]
OWN_REFERENCE = {"features": [("pw", "ffma")], "track": [("pw", "ffma"), ("corr", "ffma")]}


def all_variants(kind: str) -> List[Tuple[str, Dict[str, str]]]:
    """(name, options) of the default and every variant; kind = "features" | "track"."""
    return [("default", {})] + [(f"{k}={v}", {k: v}) for k, v in BIT_IDENTICAL + OWN_REFERENCE[kind]]


def planned(entry: str, H: int, W: int, variants, S: int) -> Dict[int, List[str]]:
    """Union of the planned batches of every option set, with the "options: launch: regime" entries each one covers."""
    out: Dict[int, List[str]] = {}
    for vname, opts in variants:
        for B, regs in plan(entry, H, W, opts, S).items():
            out.setdefault(B, []).extend(f"{vname}: {r}" for r in regs)
    return dict(sorted(out.items()))


def multi_lap(entry: str, B: int, H: int = 256, W: int = 256, opts: Optional[Dict[str, str]] = None,
              S: int = H100_SXM_SMS, **kw) -> bool:
    """Some persistent launch of the call gives a CTA at least 2 tiles at batch B."""
    return any(ln.persistent and cta_tile_counts(B * ln.tiles, S)[1] >= 2 for ln in launches(entry, H, W, opts, **kw))


# Per-frame workspace of fear_reserve (floats), in its order: bufX bufY bufE bufD, hF hT hCAT[2] hD[2] hP hQ[2], zt,
# mapB mapC, zu.  Each slot is padded to 64 floats.
K_ACT_X, K_ACT_E, K_ACT_D = 128 * 128 * 16, 128 * 128 * 96, 64 * 64 * 96
WORKSPACE_PER_FRAME = [K_ACT_X, K_ACT_X, K_ACT_E, K_ACT_D, 256 * FEAT_C, 256 * CAT_C, 256 * CAT_C, 256 * CAT_C,
                       256 * FEAT_C, 256 * FEAT_C, 256 * FEAT_C, 256 * FEAT_C, 256 * FEAT_C, TMPL_PIX * FEAT_C,
                       4 * 256, 256, TMPL_PIX * FEAT_C]


def workspace_bytes(B: int) -> int:
    return 4 * sum((pf * B + 63) // 64 * 64 for pf in WORKSPACE_PER_FRAME)


def smallest_batch_past_int32(multiple: int = 7) -> int:
    """Smallest multiple of `multiple` whose bufE (K_ACT_E floats per frame) holds more than 2^31 floats."""
    B = (2 ** 31) // K_ACT_E + 1
    return -(-B // multiple) * multiple
