"""Self-contained CPU restatement of the reference FEAR-XS inference path (ORACLE).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Plain torch CPU ops driven by a
state_dict, no nn.Module from the reference, so it travels to the GPU box where
``/root/reference`` does not exist.  ``make_golden.py`` proves it bit-identical (fp32) to the
reference's own source run through ``ref_shims`` and records golden vectors.

Every function cites the reference lines (relative to ``/root/reference``) it restates.
Pass a float64 state_dict (``to_dtype(sd, torch.float64)``) for the fp64 oracle used for
golden maps (SURVEY.md section 8(c): the fp32 CPU path is not batch-invariant).
"""
from collections import deque
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.fbnet_c import BN_EPS, FBNET_C, NUM_HOT_BLOCKS, BlockSpec

StateDict = Dict[str, torch.Tensor]

TARGET_CLASSIFICATION_KEY = "TARGET_CLASSIFICATION_KEY"  # model_training/utils/constants.py:1
TARGET_REGRESSION_LABEL_KEY = "TARGET_REGRESSION_LABEL_KEY"  # model_training/utils/constants.py:3

# model_training/config/tracker/siam_tracker.yaml:2-15
TRACKER_CONFIG = dict(
    penalty_k=0.062, window_influence=0.38, lr=0.765, windowing="cosine", total_stride=16, score_size=16,
    ratio=0.94, stride=2, bbox_ratio=0.5, template_bbox_offset=0.2, search_context=2, instance_size=256,
    template_size=128,
)
IMAGENET_MEAN = (0.485, 0.456, 0.406)  # model_training/tracker/base_tracker.py:73
IMAGENET_STD = (0.229, 0.224, 0.225)


# ------------------------------------------------------------------------------- weights
def load_lightning_state(path: str) -> StateDict:
    """model_training/utils/torch.py:11-24 -- keep keys starting with ``model.`` and strip it."""
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    return {k[len("model."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("model.")}


def to_dtype(sd: StateDict, dtype: torch.dtype) -> StateDict:
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}


def hot_path_keys(sd: StateDict) -> List[str]:
    """Keys the inference path actually reads (drops xif5_*/xif6_0/head + num_batches_tracked)."""
    dead = tuple(f"encoder.model.backbone.stages.{s.name}." for s in FBNET_C[NUM_HOT_BLOCKS:]) + (
        "encoder.model.head.",
    )
    return [k for k in sd if not k.startswith(dead) and not k.endswith("num_batches_tracked")]


# ------------------------------------------------------------------------------- layers
def _bn(sd: StateDict, prefix: str, x: torch.Tensor) -> torch.Tensor:
    """nn.BatchNorm2d in eval mode (running stats, eps 1e-5)."""
    return F.batch_norm(
        x, sd[prefix + ".running_mean"], sd[prefix + ".running_var"], sd[prefix + ".weight"], sd[prefix + ".bias"],
        False, 0.0, BN_EPS,
    )


def _conv_bn_relu(sd: StateDict, prefix: str, x, k: int, stride: int, groups: int, relu: bool) -> torch.Tensor:
    """mobile_cv ConvBNRelu: conv(bias, pad=k//2) -> BN -> ReLU (see oracle/fbnet_c.py)."""
    y = F.conv2d(x, sd[prefix + ".conv.weight"], sd[prefix + ".conv.bias"], stride, k // 2, 1, groups)
    y = _bn(sd, prefix + ".bn", y)
    return F.relu(y) if relu else y


def irf_block(sd: StateDict, prefix: str, spec: BlockSpec, x: torch.Tensor) -> torch.Tensor:
    """mobile_cv IRFBlock: [pw] -> dw -> pwl (+x)."""
    y = x
    if spec.expand != 1:
        y = _conv_bn_relu(sd, prefix + ".pw", y, 1, 1, 1, True)
    y = _conv_bn_relu(sd, prefix + ".dw", y, spec.k, spec.stride, spec.mid, True)
    y = _conv_bn_relu(sd, prefix + ".pwl", y, 1, 1, 1, False)
    return y + x if spec.residual else y


def feature_extractor(sd: StateDict, x: torch.Tensor, collect: Optional[dict] = None) -> torch.Tensor:
    """fear_net.py:58-61 + blocks.py:27-35: run fbnet_c stages 0..17 (max_layer=4)."""
    for spec in FBNET_C[:NUM_HOT_BLOCKS]:
        prefix = "encoder.model.backbone.stages." + spec.name
        if spec.kind == "conv":
            x = _conv_bn_relu(sd, prefix, x, spec.k, spec.stride, 1, True)
        elif spec.kind == "ir":
            x = irf_block(sd, prefix, spec, x)
        if collect is not None:
            collect[spec.name] = x
    return x


def neck(sd: StateDict, x: torch.Tensor) -> torch.Tensor:
    """blocks.py:75-88 AdjustLayer: conv1x1(no bias) -> BN."""
    return _bn(sd, "neck.downsample.1", F.conv2d(x, sd["neck.downsample.0.weight"]))


def get_features(sd: StateDict, crop: torch.Tensor, collect: Optional[dict] = None) -> torch.Tensor:
    """fear_net.py:63-66."""
    f = feature_extractor(sd, crop, collect)
    f = neck(sd, f)
    if collect is not None:
        collect["neck"] = f
    return f


def sep_conv(sd: StateDict, prefix: str, x: torch.Tensor) -> torch.Tensor:
    """blocks.py:45-72 SepConv(k=3, padding=1): depthwise(groups=C) -> pointwise; bias optional."""
    c = x.shape[1]
    x = F.conv2d(x, sd[prefix + ".depthwise.weight"], sd.get(prefix + ".depthwise.bias"), 1, 1, 1, c)
    return F.conv2d(x, sd[prefix + ".pointwise.weight"], sd.get(prefix + ".pointwise.bias"))


def _sep_bn_relu(sd: StateDict, seq_prefix: str, i: int, x: torch.Tensor) -> torch.Tensor:
    """One (SepConv, BN, ReLU) triple of an nn.Sequential at indices i, i+1, i+2."""
    return F.relu(_bn(sd, f"{seq_prefix}.{i + 1}", sep_conv(sd, f"{seq_prefix}.{i}", x)))


def matrix_mobile(sd: StateDict, prefix: str, z: torch.Tensor, x: torch.Tensor):
    """blocks.py:91-105: z only reshaped; x -> SepConv(bias=False)+BN+ReLU."""
    return z.reshape(z.size(0), z.size(1), -1), _sep_bn_relu(sd, prefix + ".matrix11_s", 0, x)


def pixelwise_correlation(z: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """blocks.py:121-124: s = matmul(z^T, x) viewed (b,64,w,h), then cat([x, s], dim=1)."""
    b, c, w, h = x.size()
    s = torch.matmul(z.permute(0, 2, 1), x.view(b, c, -1)).view(b, -1, w, h)
    return torch.cat([x, s], dim=1)


def mobile_correlation(sd: StateDict, prefix: str, z: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """blocks.py:108-126."""
    return _sep_bn_relu(sd, prefix + ".enc", 0, pixelwise_correlation(z, x))


def box_tower(sd: StateDict, search: torch.Tensor, kernel: torch.Tensor, update: Optional[torch.Tensor] = None,
              collect: Optional[dict] = None):
    """blocks.py:174-194 BoxTower.forward (towernum=2)."""
    p = "connect_model"
    cls_z, cls_x = matrix_mobile(sd, p + ".cls_encode", kernel if update is None else update, search)
    reg_z, reg_x = matrix_mobile(sd, p + ".reg_encode", kernel, search)
    cls_dw = mobile_correlation(sd, p + ".cls_dw", cls_z, cls_x)
    reg_dw = mobile_correlation(sd, p + ".reg_dw", reg_z, reg_x)
    x_reg = reg_dw
    for i in (0, 3):
        x_reg = _sep_bn_relu(sd, p + ".bbox_tower", i, x_reg)
    x = sd[p + ".adjust"] * sep_conv(sd, p + ".bbox_pred", x_reg) + sd[p + ".bias"]
    x = torch.exp(x)
    c = cls_dw
    for i in (0, 3):
        c = _sep_bn_relu(sd, p + ".cls_tower", i, c)
    cls = 0.1 * sep_conv(sd, p + ".cls_pred", c)
    if collect is not None:
        collect.update(cls_x=cls_x, reg_x=reg_x, cls_dw=cls_dw, reg_dw=reg_dw, x_reg=x_reg, cls_tower=c)
    return x, cls, cls_dw, x_reg


def connector(sd: StateDict, template_features: torch.Tensor, search_features: torch.Tensor,
              collect: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    """fear_net.py:76-81."""
    bbox_pred, cls_pred, _, _ = box_tower(sd, search_features, template_features, collect=collect)
    return {TARGET_REGRESSION_LABEL_KEY: bbox_pred, TARGET_CLASSIFICATION_KEY: cls_pred}


@torch.no_grad()
def forward(sd: StateDict, template: torch.Tensor, search: torch.Tensor) -> Dict[str, torch.Tensor]:
    """fear_net.py:83-88 FEARNet.forward((template, search))."""
    return connector(sd, get_features(sd, template), get_features(sd, search))


@torch.no_grad()
def track(sd: StateDict, search: torch.Tensor, template_features: torch.Tensor,
          collect: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    """fear_net.py:90-96 FEARNet.track(search, template_features)."""
    return connector(sd, template_features, get_features(sd, search, collect), collect)


# ------------------------------------------------------------------------------- decode
def make_grid(score_size: int, total_stride: int, instance_size: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """utils/utils.py:183-199: float64 (1,S,S) grids, value = (i - S//2)*stride + instance//2."""
    x, y = np.meshgrid(
        np.arange(0, score_size) - np.floor(float(score_size // 2)),
        np.arange(0, score_size) - np.floor(float(score_size // 2)),
    )
    grid_x = x * total_stride + instance_size // 2
    grid_y = y * total_stride + instance_size // 2
    return torch.from_numpy(grid_x[np.newaxis, :, :]), torch.from_numpy(grid_y[np.newaxis, :, :])


@torch.no_grad()
def decode(regression_map: torch.Tensor, classification_map: torch.Tensor, use_sigmoid: bool = True,
           config: dict = TRACKER_CONFIG):
    """dataset/box_coder.py:75-107 FEARBoxCoder.decode -> (bbox float64 (B,4) xywh, [(r,c)])."""
    grid_x, grid_y = make_grid(config["score_size"], config["total_stride"], config["instance_size"])
    if use_sigmoid:
        classification_map = classification_map.float().sigmoid()
    classification_map = classification_map[:, 0, :, :]
    pred_location = torch.stack(
        [
            grid_x - regression_map[:, 0, ...],
            grid_y - regression_map[:, 1, ...],
            grid_x + regression_map[:, 2, ...],
            grid_y + regression_map[:, 3, ...],
        ],
        dim=1,
    )
    bboxes, coords = [], []
    for one_cls, one_loc in zip(classification_map, pred_location):
        idx = int(torch.argmax(one_cls))  # first max, row-major
        r, c = idx // one_cls.shape[1], idx % one_cls.shape[1]  # utils/utils.py:175-180
        o = [m[r, c] for m in one_loc]
        bboxes.append(torch.stack([o[0], o[1], o[2] - o[0], o[3] - o[1]]))
        coords.append((r, c))
    return torch.stack(bboxes), coords


# ------------------------------------------------------------------------------- tracker
def extend_bbox(bbox, offset: float) -> np.ndarray:
    """utils/utils.py:29-57 (scalar offset form)."""
    x, y, w, h = bbox
    return np.array([x - w * offset, y - h * offset, w * (1.0 + 2 * offset), h * (1.0 + 2 * offset)]).astype("int32")


def ensure_bbox_boundaries(bbox, img_shape) -> np.ndarray:
    """utils/utils.py:60-71."""
    x1, y1, w, h = bbox
    x1, y1 = min(max(0, x1), img_shape[1]), min(max(0, y1), img_shape[0])
    x2, y2 = min(max(0, x1 + w), img_shape[1]), min(max(0, y1 + h), img_shape[0])
    return np.array([x1, y1, x2 - x1, y2 - y1]).astype("int32")


def clamp_bbox(bbox, shape, min_side: int = 3) -> np.ndarray:
    """utils/utils.py:202-212."""
    x, y, w, h = ensure_bbox_boundaries(bbox, img_shape=shape)
    img_h, img_w = shape[0], shape[1]
    if w < min_side:
        w = min_side
        x -= max(0, x + w - img_w)
    if h < min_side:
        h = min_side
        y -= max(0, y + h - img_h)
    return np.array([x, y, w, h])


def get_extended_crop(image: np.ndarray, bbox, crop_size: int, offset: float, padding_value=None):
    """utils/utils.py:215-253 with albumentations.Resize == cv2.resize(INTER_LINEAR)."""
    import cv2

    if padding_value is None:
        padding_value = np.mean(image, axis=(0, 1))
    context = extend_bbox(bbox, offset)
    pad_left, pad_top = max(-context[0], 0), max(-context[1], 0)
    pad_right = max(context[0] + context[2] - image.shape[1], 0)
    pad_bottom = max(context[1] + context[3] - image.shape[0], 0)
    crop = image[
        context[1] + pad_top: context[1] + context[3] - pad_bottom,
        context[0] + pad_left: context[0] + context[2] - pad_right,
    ]
    padded = cv2.copyMakeBorder(crop, pad_top, pad_bottom, pad_left, pad_right, cv2.BORDER_CONSTANT,
                                value=padding_value)
    padded_bbox = np.array([bbox[0] - context[0], bbox[1] - context[1], bbox[2], bbox[3]])
    padded_bbox = ensure_bbox_boundaries(padded_bbox, img_shape=padded.shape[:2])
    rows, cols = padded.shape[:2]
    if rows == crop_size and cols == crop_size:
        out = padded
    else:
        out = cv2.resize(padded, dsize=(crop_size, crop_size), interpolation=cv2.INTER_LINEAR)
    x, y, w, h = [float(v) for v in padded_bbox]
    if w * h == 0:
        raise IndexError("zero-area bbox filtered by albumentations (utils/utils.py:252)")
    x0, y0, x1, y1 = x / cols * crop_size, y / rows * crop_size, (x + w) / cols * crop_size, (y + h) / rows * crop_size
    return out, np.array([x0, y0, x1 - x0, y1 - y0]), context


def normalize_image(image: np.ndarray) -> np.ndarray:
    """base_tracker.py:69-81 albu.Normalize(imagenet): float32 (img - mean*255) * (1/(std*255))."""
    mean = np.array(IMAGENET_MEAN, dtype=np.float32)
    mean *= 255.0
    std = np.array(IMAGENET_STD, dtype=np.float32)
    std *= 255.0
    den = np.reciprocal(std, dtype=np.float32)
    img = image.astype(np.float32)
    img -= mean
    img *= den
    return img


def preprocess_image(image: np.ndarray) -> torch.Tensor:
    """base_tracker.py:97-103 (3-channel case): normalise, HWC -> 1CHW float32."""
    img = normalize_image(image[:, :, :3])
    return torch.from_numpy(np.expand_dims(np.transpose(img, (2, 0, 1)), 0)).float()


def rescale_bbox(bbox: np.ndarray, padded_box, instance_size: int = 256) -> List[int]:
    """base_tracker.py:83-90 (python round(); sides >= 3)."""
    w_scale = padded_box[2] / instance_size
    h_scale = padded_box[3] / instance_size
    bbox = list(bbox)
    bbox[0] = round(bbox[0] * w_scale + padded_box[0])
    bbox[1] = round(bbox[1] * h_scale + padded_box[1])
    bbox[2] = max(3, round(bbox[2] * w_scale))
    bbox[3] = max(3, round(bbox[3] * h_scale))
    return list(map(int, bbox))


def limit(radius):
    """utils/utils.py:74-77."""
    if isinstance(radius, torch.Tensor):
        return torch.maximum(radius, 1.0 / radius)
    return np.maximum(radius, 1.0 / radius)


def squared_size(w, h):
    """utils/utils.py:80-85."""
    pad = (w + h) * 0.5
    size = (w + pad) * (h + pad)
    if isinstance(size, torch.Tensor):
        return torch.sqrt(size)
    return np.sqrt(size)


def tracking_window(windowing: str, score_size: int) -> torch.Tensor:
    """base_tracker.py:57-67."""
    if windowing == "cosine":
        return torch.from_numpy(np.outer(np.hanning(score_size), np.hanning(score_size)))
    return torch.ones(int(score_size), int(score_size))


def confidence_postprocess(cls_score: torch.Tensor, regression_map: torch.Tensor, prev_size, window: torch.Tensor,
                           config: dict):
    """base_tracker.py:166-205 with ``smooth: true``: scale / ratio penalty and cosine-window re-weighting of the
    score map.  cls_score (1,1,16,16) float32 (sigmoid applied), regression_map (1,4,16,16) -> (pscore, penalty)."""
    grid_x, grid_y = make_grid(config["score_size"], config["total_stride"], config["instance_size"])
    pred_location = torch.stack(
        [grid_x - regression_map[:, 0, ...], grid_y - regression_map[:, 1, ...],
         grid_x + regression_map[:, 2, ...], grid_y + regression_map[:, 3, ...]], dim=1)[0]
    s_c = limit(squared_size(pred_location[2] - pred_location[0], pred_location[3] - pred_location[1])
                / (squared_size(prev_size[0], prev_size[1])))
    r_c = limit((prev_size[0] / prev_size[1])
                / ((pred_location[2] - pred_location[0]) / (pred_location[3] - pred_location[1])))
    penalty = torch.exp(-(r_c * s_c - 1) * config["penalty_k"])
    pscore = penalty * cls_score
    pscore = pscore * (1 - config["window_influence"]) + window * config["window_influence"]
    return pscore, penalty.cpu().numpy()


def smooth_size(size: np.ndarray, prev_size: np.ndarray, lr: float):
    """base_tracker.py:126-139."""
    size = size * lr
    prev_size = prev_size * (1 - lr)
    w = prev_size[0] + lr * (size[0] + prev_size[0])
    h = prev_size[1] + lr * (size[1] + prev_size[1])
    return w, h


class OracleTracker:
    """fear_tracker.py:13-86 + base_tracker.py:28-205.  With the default config (no ``smooth`` key)
    _confidence_postprocess / _postprocess_bbox are pass-throughs (base_tracker.py:152,174); ``smooth=True`` in the
    config enables the penalty / window / size-smoothing branch."""

    def __init__(self, sd: StateDict, config: dict = TRACKER_CONFIG):
        self.sd, self.cfg = sd, dict(config)
        self.dtype = sd["neck.downsample.0.weight"].dtype
        self.bbox = None
        self.mean_color = None
        self.template_features = None
        self.paths = None
        self.prev_size = None
        self.last_search_crop = None
        self.last_maps = None
        self.window = tracking_window(self.cfg["windowing"], self.cfg["score_size"])

    def initialize(self, image: np.ndarray, rect) -> None:
        rect = clamp_bbox(rect, image.shape)
        self.bbox = rect
        self.paths = deque([rect], maxlen=10)
        self.mean_color = np.mean(image, axis=(0, 1))
        crop, _, _ = get_extended_crop(image, rect, self.cfg["template_size"], self.cfg["template_bbox_offset"])
        self.template_crop = crop
        with torch.no_grad():
            self.template_features = get_features(self.sd, preprocess_image(crop).to(self.dtype))

    def postprocess(self, out):
        """FEARTracker._postprocess (fear_tracker.py:74-86) on a maps dictionary."""
        cls_score = out[TARGET_CLASSIFICATION_KEY].detach().float().sigmoid()
        regression_map = out[TARGET_REGRESSION_LABEL_KEY].detach().float()
        penalty = None
        classification_map = cls_score
        if self.cfg.get("smooth", False):
            classification_map, penalty = confidence_postprocess(cls_score, regression_map, self.prev_size, self.window,
                                                                 self.cfg)
        bbox, coords = decode(out[TARGET_REGRESSION_LABEL_KEY], classification_map, use_sigmoid=False, config=self.cfg)
        r, c = coords[0]
        cls_np = np.squeeze(cls_score)
        pred_bbox = np.squeeze(bbox.cpu().numpy())
        if self.cfg.get("smooth", False):  # _postprocess_bbox, base_tracker.py:147-164
            lr = (penalty[r, c] * cls_np[r, c] * self.cfg["lr"]).item()
            pred_w, pred_h = smooth_size(np.array(pred_bbox[2:]), prev_size=self.prev_size, lr=lr)
            pred_bbox = np.array([pred_bbox[0], pred_bbox[1], pred_w, pred_h])
        return pred_bbox, cls_np[r, c], (r, c)

    def track(self, search_crop: np.ndarray):
        out = track(self.sd, preprocess_image(search_crop).to(self.dtype), self.template_features)
        self.last_maps = out
        return self.postprocess(out)

    def update(self, image: np.ndarray) -> Dict[str, np.ndarray]:
        crop, search_bbox, padded = get_extended_crop(
            image, self.bbox, self.cfg["instance_size"], self.cfg["search_context"], self.mean_color)
        self.last_search_crop = crop
        self.prev_size = search_bbox[2:]
        pred, _, _ = self.track(crop)
        pred = rescale_bbox(pred, padded, self.cfg["instance_size"])
        pred = clamp_bbox(pred, image.shape)
        self.bbox = pred
        self.paths.append(pred)
        return dict(bbox=pred)


def read_video_rgb(path: str) -> np.ndarray:
    """demo_video.py:53 reads with imageio (absent here) -> cv2 decode + BGR->RGB."""
    import cv2

    cap = cv2.VideoCapture(path)
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    cap.release()
    return np.stack(frames)


# ------------------------------------------------------------------------------- inputs
def synthetic_crops(batch: int, seed: int = 20260924, with_template: bool = True):
    """SURVEY.md section 8(d): uniform uint8 crops, templates drawn first then searches,
    ImageNet-normalised with the tracker's float32 arithmetic.  Returns (template, search)
    float32 NCHW tensors plus the raw uint8 arrays."""
    g = torch.Generator().manual_seed(seed)
    zu = torch.randint(0, 256, (batch, 3, 128, 128), generator=g, dtype=torch.uint8)
    xu = torch.randint(0, 256, (batch, 3, 256, 256), generator=g, dtype=torch.uint8)

    def norm(u):
        hwc = u.permute(0, 2, 3, 1).numpy()
        return torch.from_numpy(np.stack([normalize_image(i) for i in hwc])).permute(0, 3, 1, 2).contiguous()

    return (norm(zu) if with_template else None), norm(xu), zu, xu


def shape_crops(h: int, w: int, batch: int, seed: int = 11):
    """Seeded uniform uint8 crops of any size (H, W), ImageNet-normalised as in synthetic_crops.
    Returns (float32 NCHW, uint8 NCHW)."""
    g = torch.Generator().manual_seed(seed * 100003 + h * 1009 + w)
    u = torch.randint(0, 256, (batch, 3, h, w), generator=g, dtype=torch.uint8)
    hwc = u.permute(0, 2, 3, 1).numpy()
    x = torch.from_numpy(np.stack([normalize_image(i) for i in hwc])).permute(0, 3, 1, 2).contiguous()
    return x, u
