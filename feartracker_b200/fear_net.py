"""FEARNet with the reference's Python API, executed by libfear_b200 (sm_90a CUDA kernels).

Drop-in for ``model_training.model.fear_net.FEARNet`` (reference fear_net.py:14-96): same
constructor keywords (extras swallowed by ``**kwargs`` because hydra passes every YAML key),
same sub-module / parameter names so ``load_state_dict(strict=True)`` of the shipped Lightning
checkpoint works, same methods and output dictionary.  The nn.Module tree below only HOLDS
parameters; arithmetic never runs in PyTorch.  On first use in eval mode the parameters are
BN-folded (float64) and packed into the library; ``load_state_dict`` / ``train()`` / ``.to`` /
``.cuda`` invalidate the packed copy.  Eval mode has no CPU path (non-CUDA inputs raise).  In ``train()`` mode
(BatchNorm batch statistics + autograd, which the inference kernels do not provide) the same methods run the plain
PyTorch graph of ``torch_graph.py`` over the same parameters -- NOT accelerated; it exists so the reference's training
step (``FEARLightningModel.forward`` -> ``model.forward``, fear_lightning_model.py:60-62) runs on this class.
"""
import ctypes
import weakref
from collections import OrderedDict
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib, torch_graph, weights
from .constants import TARGET_CLASSIFICATION_KEY, TARGET_REGRESSION_LABEL_KEY

# (name, cin, cout, kernel, stride, expansion) of fbnet_c's 24 stages; expansion None = plain
# conv-bn(-relu), "skip" = identity.  Channel / kernel numbers are those of the checkpoint.
_FBNET_C_STAGES = (
    ("xif0_0", 3, 16, 3, 2, None), ("xif1_0", 16, 16, 3, 1, 1), ("xif2_0", 16, 24, 3, 2, 6),
    ("xif2_1", 24, 24, 0, 1, "skip"), ("xif2_2", 24, 24, 3, 1, 1), ("xif2_3", 24, 24, 3, 1, 1),
    ("xif3_0", 24, 32, 5, 2, 6), ("xif3_1", 32, 32, 5, 1, 3), ("xif3_2", 32, 32, 5, 1, 6),
    ("xif3_3", 32, 32, 3, 1, 6), ("xif4_0", 32, 64, 5, 2, 6), ("xif4_1", 64, 64, 5, 1, 3),
    ("xif4_2", 64, 64, 5, 1, 6), ("xif4_3", 64, 64, 5, 1, 6), ("xif4_4", 64, 112, 5, 1, 6),
    ("xif4_5", 112, 112, 5, 1, 6), ("xif4_6", 112, 112, 5, 1, 6), ("xif4_7", 112, 112, 5, 1, 3),
    ("xif5_0", 112, 184, 5, 2, 6), ("xif5_1", 184, 184, 5, 1, 6), ("xif5_2", 184, 184, 5, 1, 6),
    ("xif5_3", 184, 184, 5, 1, 6), ("xif5_4", 184, 352, 3, 1, 6), ("xif6_0", 352, 1984, 1, 1, None),
)


class _Params(nn.Module):
    """A module that only stores parameters; calling it is an error (the library does the math)."""

    def forward(self, *args, **kwargs):
        raise RuntimeError(
            f"{type(self).__name__} is a parameter container of the H100 FEARNet; call FEARNet.forward / "
            "track / get_features (executed by libfear_b200) instead"
        )


class _ConvBN(_Params):
    def __init__(self, cin, cout, k, stride, groups=1):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, groups=groups, bias=True)
        self.bn = nn.BatchNorm2d(cout)


class _IRF(_Params):
    def __init__(self, cin, cout, k, stride, expansion):
        super().__init__()
        mid = cin * expansion
        if expansion != 1:
            self.pw = _ConvBN(cin, mid, 1, 1)
        self.dw = _ConvBN(mid, mid, k, stride, groups=mid)
        self.pwl = _ConvBN(mid, cout, 1, 1)


class _Sep(_Params):
    """depthwise 3x3 + pointwise 1x1 pair (names as in the checkpoint)."""

    def __init__(self, cin, cout, bias=True):
        super().__init__()
        self.depthwise = nn.Conv2d(cin, cin, 3, padding=1, groups=cin, bias=bias)
        self.pointwise = nn.Conv2d(cin, cout, 1, bias=bias)


class _FBNetC(_Params):
    def __init__(self):
        super().__init__()
        stages = OrderedDict()
        for name, cin, cout, k, stride, e in _FBNET_C_STAGES:
            if e == "skip":
                stages[name] = nn.Identity()
            elif e is None:
                stages[name] = _ConvBN(cin, cout, k, stride)
            else:
                stages[name] = _IRF(cin, cout, k, stride, e)
        self.backbone = _Params()
        self.backbone.stages = nn.Sequential(stages)
        self.head = _Params()
        self.head.conv = nn.Conv2d(1984, 1000, 1)


class Encoder(_Params):
    """Parameter container with the attribute surface of the reference Encoder (blocks.py:8-42)."""

    encoder_channels = {"layer0": 352, "layer1": 112, "layer2": 32, "layer3": 24, "layer4": 16}

    def __init__(self, pretrained: bool = True):
        super().__init__()
        self.pretrained = pretrained  # never downloads: the FEAR checkpoint overwrites everything
        self.model = _FBNetC()
        s = self.model.backbone.stages
        self.stages = [s[:2], s[2:5], s[5:9], s[9:18], s[18:23]]


class AdjustLayer(_Params):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.downsample = nn.Sequential(nn.Conv2d(in_channels, out_channels, 1, bias=False),
                                        nn.BatchNorm2d(out_channels))


def _sep_bn_relu(cin, cout, bias=True):
    return nn.Sequential(_Sep(cin, cout, bias=bias), nn.BatchNorm2d(cout), nn.ReLU(inplace=True))


class _SeqHolder(_Params):
    def __init__(self, attr, seq):
        super().__init__()
        setattr(self, attr, seq)


class BoxTower(_Params):
    """Parameter container for the reference BoxTower (blocks.py:129-172), towernum = 2.
    Calling it runs the library head and returns the reference's 4-tuple
    ``(bbox, cls, cls_dw, x_reg)`` (blocks.py:174-194)."""

    _owner = None  # weakref to the FEARNet that executes this tower

    def forward(self, search, kernel, update=None):
        owner = self._owner() if self._owner is not None else None
        if owner is None:
            return super().forward()
        if owner.training:
            return torch_graph.box_tower(owner, search, kernel, update)
        out = owner._head(kernel, search, update)  # update: dynamic template of the cls branch (blocks.py:174-179)
        b = search.shape[0]
        return (out[TARGET_REGRESSION_LABEL_KEY], out[TARGET_CLASSIFICATION_KEY],
                owner.head_tensor("cls_dw", b), owner.head_tensor("x_reg", b))

    def __init__(self, channels: int = 256, corr_channels: int = 64, towernum: int = 2):
        super().__init__()
        self.cls_encode = _SeqHolder("matrix11_s", _sep_bn_relu(channels, channels, bias=False))
        self.reg_encode = _SeqHolder("matrix11_s", _sep_bn_relu(channels, channels, bias=False))
        self.cls_dw = _SeqHolder("enc", _sep_bn_relu(channels + corr_channels, channels))
        self.reg_dw = _SeqHolder("enc", _sep_bn_relu(channels + corr_channels, channels))
        for name in ("bbox_tower", "cls_tower"):
            layers = []
            for _ in range(towernum):
                layers += [_Sep(channels, channels), nn.BatchNorm2d(channels), nn.ReLU()]
            self.add_module(name, nn.Sequential(*layers))
        self.bbox_pred = _Sep(channels, 4)
        self.cls_pred = _Sep(channels, 1)
        self.adjust = nn.Parameter(0.1 * torch.ones(1))
        self.bias = nn.Parameter(torch.ones(1, 4, 1, 1))


def _make_grid(score_size: int, total_stride: int, instance_size: int):
    """float64 (1,S,S) pixel-centre grids: (i - S//2) * stride + instance//2 (reference
    utils/utils.py:183-199)."""
    ax = (np.arange(score_size, dtype=np.float64) - float(score_size // 2)) * total_stride + instance_size // 2
    gx, gy = np.meshgrid(ax, ax)
    return torch.from_numpy(gx[None]), torch.from_numpy(gy[None])


class FEARNet(nn.Module):
    def __init__(
        self,
        backbone=None,
        img_size: int = 256,
        pretrained: bool = True,
        score_size: int = 25,
        adjust_channels: int = 256,
        total_stride: int = 8,
        instance_size: int = 255,
        towernum: int = 4,
        max_layer: int = 3,
        crop_template_features: bool = True,
        conv_block: str = "regular",
        mobile: bool = False,
        **kwargs,
    ) -> None:
        assert max_layer in (3, 4)  # reference fear_net.py:31-32
        super().__init__()
        if max_layer != 4 or towernum != 2 or adjust_channels != 256:
            raise NotImplementedError(
                "libfear_b200 implements the FEAR-XS configuration only (max_layer=4, towernum=2, "
                f"adjust_channels=256 -- model_training/config/model/fear.yaml); got max_layer={max_layer}, "
                f"towernum={towernum}, adjust_channels={adjust_channels}"
            )
        self.encoder = Encoder(pretrained)
        self.neck = AdjustLayer(self.encoder.encoder_channels["layer1"], adjust_channels)
        self.connect_model = BoxTower(adjust_channels, 64, towernum)
        object.__setattr__(self.connect_model, "_owner", weakref.ref(self))
        self.search_size = img_size
        self.score_size = score_size
        self.total_stride = total_stride
        self.instance_size = instance_size
        self.size = 1
        self.max_layer = max_layer
        self.crop_template_features = crop_template_features
        self.features = None
        self.grid_x = torch.empty(0)
        self.grid_y = torch.empty(0)
        self.grids(self.size)
        self._handle: Optional[ctypes.c_void_p] = None
        self._handle_device: Optional[int] = None
        self._reserved = 0

    # ------------------------------------------------------------------ reference surface
    def grids(self, size: int) -> None:
        gx, gy = _make_grid(self.score_size, self.total_stride, self.instance_size)
        self.grid_x, self.grid_y = gx.unsqueeze(0).repeat(size, 1, 1, 1), gy.unsqueeze(0).repeat(size, 1, 1, 1)

    def feature_extractor(self, x: torch.Tensor) -> torch.Tensor:
        """(B,3,H,W) -> (B,112,H/16,W/16): fbnet_c stages 0..17."""
        if self.training:
            return torch_graph.feature_extractor(self, x)
        x, h, lib = self._prep(x)
        b, _, hh, ww = x.shape
        out = torch.empty((b, 112, hh // 16, ww // 16), device=x.device, dtype=torch.float32)
        _lib.check(lib.fear_backbone(h, x.data_ptr(), b, hh, ww, out.data_ptr(), self._stream(x)), "fear_backbone")
        return out

    def get_features(self, crop: torch.Tensor) -> torch.Tensor:
        """(B,3,H,W) float -> (B,256,H/16,W/16).  A uint8 (B,H,W,3) RGB crop is also accepted: it is
        ImageNet-normalised inside the stem kernel (bit-identical to Tracker._preprocess_image on the host)."""
        if self.training:
            return torch_graph.get_features(self, crop)
        if crop.dtype == torch.uint8:
            x, h, lib = self._prep(crop, keep_dtype=True)
            b, hh, ww, ch = x.shape
            if ch != 3:
                raise ValueError(f"uint8 crops must be (B,H,W,3), got {tuple(x.shape)}")
            out = torch.empty((b, 256, hh // 16, ww // 16), device=x.device, dtype=torch.float32)
            _lib.check(lib.fear_get_features_u8(h, x.data_ptr(), b, hh, ww, out.data_ptr(), self._stream(x)),
                       "fear_get_features_u8")
            return out
        x, h, lib = self._prep(crop)
        b, _, hh, ww = x.shape
        out = torch.empty((b, 256, hh // 16, ww // 16), device=x.device, dtype=torch.float32)
        _lib.check(lib.fear_get_features(h, x.data_ptr(), b, hh, ww, out.data_ptr(), self._stream(x)),
                   "fear_get_features")
        return out

    def connector(self, template_features: torch.Tensor, search_features: torch.Tensor) -> Dict[str, torch.Tensor]:
        if self.training:
            return torch_graph.connector(self, template_features, search_features)
        return self._head(template_features, search_features, None)

    def _head(self, template_features: torch.Tensor, search_features: torch.Tensor,
              update: Optional[torch.Tensor]) -> Dict[str, torch.Tensor]:
        """BoxTower.forward(search, kernel, update) in the library (fear_head_update); update = None is the
        reference's only call pattern (fear_net.py:77)."""
        xf, h, lib = self._prep(search_features)
        zf = self._as_input(template_features, xf.device)
        b = xf.shape[0]
        self._check_shapes(zf, b)
        zu = None
        if update is not None:
            zu = self._as_input(update, xf.device)
            self._check_shapes(zu, b)
        if tuple(xf.shape[1:]) != (256, 16, 16):
            raise ValueError(f"search features must be (B,256,16,16), got {tuple(xf.shape)}")
        bbox = torch.empty((b, 4, 16, 16), device=xf.device, dtype=torch.float32)
        cls = torch.empty((b, 1, 16, 16), device=xf.device, dtype=torch.float32)
        _lib.check(lib.fear_head_update(h, zf.data_ptr(), zf.shape[0], zu.data_ptr() if zu is not None else None,
                                        zu.shape[0] if zu is not None else 0, xf.data_ptr(), b, bbox.data_ptr(),
                                        cls.data_ptr(), self._stream(xf)), "fear_head_update")
        return {TARGET_REGRESSION_LABEL_KEY: bbox, TARGET_CLASSIFICATION_KEY: cls}

    def forward(self, x: Tuple[torch.Tensor, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.training:
            return torch_graph.forward(self, x)
        template, search = x
        s, h, lib = self._prep(search)
        t = self._as_input(template, s.device)
        b = s.shape[0]
        self.size = b
        if tuple(t.shape) != (b, 3, 128, 128) or tuple(s.shape) != (b, 3, 256, 256):
            raise ValueError(f"forward expects template (B,3,128,128) and search (B,3,256,256); got "
                             f"{tuple(t.shape)} / {tuple(s.shape)}")
        bbox = torch.empty((b, 4, 16, 16), device=s.device, dtype=torch.float32)
        cls = torch.empty((b, 1, 16, 16), device=s.device, dtype=torch.float32)
        _lib.check(lib.fear_forward(h, t.data_ptr(), s.data_ptr(), b, bbox.data_ptr(), cls.data_ptr(), None,
                                    self._stream(s)), "fear_forward")
        return {TARGET_REGRESSION_LABEL_KEY: bbox, TARGET_CLASSIFICATION_KEY: cls}

    def track(self, search: torch.Tensor, template_features: torch.Tensor) -> Dict[str, torch.Tensor]:
        if self.training:
            return torch_graph.track(self, search, template_features)
        out, _ = self._track(search, template_features, want_maps=True, want_boxes=False)
        return out

    # ------------------------------------------------------------------ extensions
    def track_boxes(self, search: torch.Tensor, template_features: torch.Tensor, with_maps: bool = False):
        """track() + on-device FEARBoxCoder.decode.  Returns a uint8 tensor (B,48) of FearBox records
        (view with ``boxes_to_numpy``) and, if requested, the maps dictionary."""
        maps, boxes = self._track(search, template_features, want_maps=with_maps, want_boxes=True)
        return (boxes, maps) if with_maps else boxes

    def track_boxes_from_host(self, search_host: torch.Tensor, template_features_host: torch.Tensor,
                              out_host: Optional[torch.Tensor] = None, chunks: int = 1) -> torch.Tensor:
        """End-to-end batched call on PINNED host buffers (uint8 (B,256,256,3) raw crops or float32
        (B,3,256,256) normalised crops, plus float32 template features).

        The host->device copies run on a side stream into one of TWO staging sets, so the copy of call i+1
        overlaps the kernels of call i (and, with ``chunks`` > 1, the copy of slice j+1 overlaps the kernels
        of slice j inside one call).  The 48-byte box records of the whole batch are copied back to
        ``out_host`` if given.  No host synchronisation: synchronise the current stream (or an event) before
        reading ``out_host`` / the returned device tensor, which stays valid until the call after next."""
        dev = next(self.parameters()).device
        if self.training or dev.type != "cuda":
            raise RuntimeError("track_boxes_from_host needs the model in eval mode on a CUDA device")
        b = search_host.shape[0]
        bz = template_features_host.shape[0]
        chunks = max(1, min(chunks, b))
        comp = torch.cuda.current_stream(dev)
        if getattr(self, "_copy_stream", None) is None or self._copy_stream.device != dev:
            self._copy_stream = torch.cuda.Stream(dev)
            self._stage, self._stage_key, self._stage_flip = None, None, 0
        key = (b, bz, chunks, search_host.dtype, tuple(search_host.shape[1:]))
        if self._stage_key != key:
            bounds = [(i * b // chunks, (i + 1) * b // chunks) for i in range(chunks)]

            def make_set():
                return dict(
                    x=[torch.empty((e - s,) + tuple(search_host.shape[1:]), device=dev, dtype=search_host.dtype)
                       for s, e in bounds],
                    z=torch.empty((bz, 256, 8, 8), device=dev),
                    boxes=torch.empty((b, _lib.BOX_DTYPE.itemsize), device=dev, dtype=torch.uint8),
                    ready=[torch.cuda.Event() for _ in bounds], zready=torch.cuda.Event(), free=torch.cuda.Event())

            self._stage = dict(bounds=bounds, sets=[make_set(), make_set()])
            self._stage_key, self._stage_flip = key, 0
            for st in self._stage["sets"]:
                st["free"].record(comp)
        st = self._stage["sets"][self._stage_flip]
        self._stage_flip ^= 1
        bounds = self._stage["bounds"]
        copy = self._copy_stream
        copy.wait_event(st["free"])  # kernels of the call that last used this staging set have finished
        with torch.cuda.stream(copy):
            st["z"].copy_(template_features_host, non_blocking=True)
            st["zready"].record(copy)
            for i, (s0, e0) in enumerate(bounds):
                st["x"][i].copy_(search_host[s0:e0], non_blocking=True)
                st["ready"][i].record(copy)
        comp.wait_event(st["zready"])
        for i, (s0, e0) in enumerate(bounds):
            comp.wait_event(st["ready"][i])
            zf = st["z"] if bz == 1 else st["z"][s0:e0]
            if chunks == 1:
                st["boxes"] = self.track_boxes(st["x"][i], zf)
            else:
                st["boxes"][s0:e0] = self.track_boxes(st["x"][i], zf)
        st["free"].record(comp)
        if out_host is not None:
            out_host.copy_(st["boxes"], non_blocking=True)
        return st["boxes"]

    @staticmethod
    def boxes_to_numpy(boxes: torch.Tensor) -> np.ndarray:
        return boxes.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)

    def head_tensor(self, name: str, batch: int) -> torch.Tensor:
        """NCHW copy of a head intermediate of the last call: "cat_cls" | "cat_reg" (B,320,16,16);
        "search_features" | "cls_dw" | "reg_dw" | "x_reg" | "cls_tower" (B,256,16,16)."""
        dev = next(self.parameters()).device
        h, lib = self._ensure_handle(dev)
        ch = 320 if name.startswith("cat_") else 256
        out = torch.empty((batch, ch, 16, 16), device=dev, dtype=torch.float32)
        _lib.check(lib.fear_debug_head_tensor(h, name.encode(), batch, out.data_ptr(),
                                              torch.cuda.current_stream(dev).cuda_stream), "fear_debug_head_tensor")
        return out

    def backbone_prefix(self, img: torch.Tensor, nblocks: int) -> torch.Tensor:
        """Debug: activation after the stem + first ``nblocks`` backbone blocks, NCHW."""
        x, h, lib = self._prep(img)
        chans = [16] + [c for (_, _, c, _, _, e) in _FBNET_C_STAGES[1:18] if e != "skip"]
        strides = [2] + [s for (_, _, _, _, s, e) in _FBNET_C_STAGES[1:18] if e != "skip"]
        down = int(np.prod(strides[: nblocks + 1]))
        b, _, hh, ww = x.shape
        out = torch.empty((b, chans[nblocks], hh // down, ww // down), device=x.device, dtype=torch.float32)
        _lib.check(lib.fear_debug_backbone_prefix(h, x.data_ptr(), b, hh, ww, nblocks, out.data_ptr(),
                                                  self._stream(x)), "fear_debug_backbone_prefix")
        return out

    def reserve(self, max_batch: int) -> None:
        """Pre-allocate library workspace for batches up to ``max_batch`` (larger batches are chunked)."""
        self._reserved = max(self._reserved, int(max_batch))
        if self._handle is not None:
            _lib.check(_lib.load().fear_reserve(self._handle, self._reserved), "fear_reserve")

    def set_option(self, key: str, value: str) -> None:
        dev = next(self.parameters()).device
        h, lib = self._ensure_handle(dev)
        _lib.check(lib.fear_set_option(h, key.encode(), value.encode()), "fear_set_option")

    def generation(self):
        """Changes whenever CUDA-graph captures of calls on this net go stale: weights re-packed (new handle),
        workspace re-allocated by a larger ``reserve`` / batch, or an option changed."""
        if self._handle is None:
            return None
        return (self._handle.value, int(_lib.load().fear_generation(self._handle)))

    def launch_count(self) -> int:
        return int(_lib.load().fear_launch_count(self._handle)) if self._handle is not None else 0

    def profile(self, enable: bool) -> None:
        dev = next(self.parameters()).device
        h, lib = self._ensure_handle(dev)
        _lib.check(lib.fear_profile(h, int(enable)), "fear_profile")

    def stage_times(self) -> Dict[str, Tuple[float, int]]:
        lib = _lib.load()
        out = {}
        for i, name in enumerate(_lib.stage_names()):
            ms, n = ctypes.c_float(), ctypes.c_int64()
            _lib.check(lib.fear_stage_ms(self._handle, i, ctypes.byref(ms), ctypes.byref(n)), "fear_stage_ms")
            out[name] = (ms.value, n.value)
        return out

    # ------------------------------------------------------------------ internals
    def _track(self, search, template_features, want_maps: bool, want_boxes: bool):
        u8 = search.dtype == torch.uint8
        s, h, lib = self._prep(search, keep_dtype=u8)
        zf = self._as_input(template_features, s.device)
        b = s.shape[0]
        self._check_shapes(zf, b)
        if tuple(s.shape[1:]) != ((256, 256, 3) if u8 else (3, 256, 256)):
            raise ValueError(f"search must be float (B,3,256,256) or uint8 (B,256,256,3), got {tuple(s.shape)}")
        bbox = cls = boxes = None
        if want_maps:
            bbox = torch.empty((b, 4, 16, 16), device=s.device, dtype=torch.float32)
            cls = torch.empty((b, 1, 16, 16), device=s.device, dtype=torch.float32)
        if want_boxes:
            boxes = torch.empty((b, _lib.BOX_DTYPE.itemsize), device=s.device, dtype=torch.uint8)
        entry = lib.fear_track_u8 if u8 else lib.fear_track
        _lib.check(
            entry(h, s.data_ptr(), zf.data_ptr(), zf.shape[0], b,
                           bbox.data_ptr() if want_maps else None, cls.data_ptr() if want_maps else None,
                           boxes.data_ptr() if want_boxes else None, self._stream(s)),
            "fear_track")
        maps = {TARGET_REGRESSION_LABEL_KEY: bbox, TARGET_CLASSIFICATION_KEY: cls} if want_maps else None
        return maps, boxes

    @staticmethod
    def _check_shapes(zf: torch.Tensor, b: int) -> None:
        if tuple(zf.shape[1:]) != (256, 8, 8) or zf.shape[0] not in (1, b):
            raise ValueError(f"template features must be (B|1,256,8,8) for batch {b}, got {tuple(zf.shape)}")

    @staticmethod
    def _stream(t: torch.Tensor) -> int:
        return torch.cuda.current_stream(t.device).cuda_stream

    @staticmethod
    def _as_input(t: torch.Tensor, device: torch.device) -> torch.Tensor:
        if t.device != device:
            raise ValueError(f"all inputs must live on {device}, got {t.device}")
        return t.detach().to(torch.float32).contiguous()

    def _prep(self, x: torch.Tensor, keep_dtype: bool = False):
        if self.training:
            raise RuntimeError("internal: the library path was entered in train() mode")
        if not x.is_cuda:
            raise RuntimeError("FEARNet (H100) has no CPU path: inputs must be CUDA tensors on an H100 (sm_90)")
        x = x.detach().contiguous() if keep_dtype else self._as_input(x, x.device)
        h, lib = self._ensure_handle(x.device)
        if x.shape[0] > self._reserved:
            self.reserve(x.shape[0])
        return x, h, lib

    def _ensure_handle(self, device: torch.device):
        if device.type != "cuda":
            raise RuntimeError("FEARNet (H100) needs a CUDA device")
        index = device.index if device.index is not None else torch.cuda.current_device()
        if self._handle is not None and self._handle_device == index:
            return self._handle, _lib.load()
        self._drop_handle()
        sd = {k: v for k, v in self.state_dict().items() if v.is_floating_point()}
        with torch.cuda.device(index):  # the handle belongs to the device current at pack time; caller's is restored
            lib = _lib.init(index)
            blob, offsets = weights.pack(sd, _lib.weight_table())
            handle = ctypes.c_void_p()
            _lib.check(
                lib.fear_pack_weights(blob.ctypes.data_as(ctypes.c_void_p),
                                      offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), len(offsets) - 1,
                                      ctypes.byref(handle)),
                "fear_pack_weights")
            self._handle, self._handle_device = handle, index
            if self._reserved > 1:
                _lib.check(lib.fear_reserve(handle, self._reserved), "fear_reserve")
        return handle, lib

    def _drop_handle(self) -> None:
        if getattr(self, "_handle", None) is not None:
            _lib.load().fear_free(self._handle)
        self._handle, self._handle_device = None, None

    def load_state_dict(self, *args, **kwargs):
        self._drop_handle()
        return super().load_state_dict(*args, **kwargs)

    def train(self, mode: bool = True):
        # the packed copy only goes stale when parameters can change, i.e. on entering train(); eval() -> eval()
        # (a common per-sequence idiom) keeps the handle, its workspace and any captured CUDA graph
        if mode:
            self._drop_handle()
        return super().train(mode)

    def _apply(self, fn, *args, **kwargs):
        self._drop_handle()
        return super()._apply(fn, *args, **kwargs)

    def __del__(self):
        try:
            self._drop_handle()
        except Exception:
            pass
