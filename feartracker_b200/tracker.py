"""FEARTracker: stateful single-object tracker around the H100 FEARNet.

API mirror of reference model_training/tracker/base_tracker.py:28-124 and fear_tracker.py:13-86:
``FEARTracker(model, cuda_id=0, **tracking_config)``, ``initialize(image, rect)``,
``update(image) -> {"bbox": [x, y, w, h]}``, ``track(search_crop)``, ``get_template_features``,
``to_device``, ``reset``.  Cropping / normalisation stay on the host (cv2 fixed-point resize is part
of the reference's observable behaviour); network + decode run in libfear_b200 and only the
48-byte box record comes back per frame.
"""
from collections import deque
from typing import Any, Dict, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn as nn

from . import image_ops
from .box_coder import FEARBoxCoder, TrackerDecodeResult
from .constants import TARGET_CLASSIFICATION_KEY, TARGET_REGRESSION_LABEL_KEY


class TrackingState:
    def __init__(self) -> None:
        self.frame_h = 0
        self.frame_w = 0
        self.bbox: Optional[np.ndarray] = None
        self.mapping: Optional[np.ndarray] = None
        self.prev_size = None
        self.mean_color = None
        self.paths = None

    def save_frame_shape(self, frame: np.ndarray) -> None:
        self.frame_h, self.frame_w = frame.shape[0], frame.shape[1]


class Tracker:
    def __init__(self, model: nn.Module, cuda_id: Union[int, str] = 0, **tracking_config: Any) -> None:
        self.cuda_id = cuda_id
        self.tracking_config = tracking_config
        self.tracking_state = TrackingState()
        self.net = model
        self.box_coder = self.get_box_coder(tracking_config, cuda_id)
        self._template_features = None
        self.window = self._get_tracking_window(tracking_config["windowing"], tracking_config["score_size"])
        self.to_device(cuda_id)

    def get_box_coder(self, tracking_config, cuda_id: int = 0):
        raise NotImplementedError

    def to_device(self, cuda_id) -> None:
        self.cuda_id = cuda_id
        self.box_coder = self.box_coder.to_device(cuda_id)

    @staticmethod
    def _get_tracking_window(windowing: str, score_size: int) -> np.ndarray:
        if windowing == "cosine":
            return np.outer(np.hanning(score_size), np.hanning(score_size))
        return np.ones((int(score_size), int(score_size)))

    def _device(self) -> torch.device:
        if not torch.cuda.is_available():
            raise RuntimeError("FEARTracker (H100) needs a CUDA device: there is no CPU path")
        if isinstance(self.cuda_id, int):
            return torch.device("cuda", self.cuda_id)
        dev = torch.device(self.cuda_id)  # the reference also takes device strings ("cuda:1")
        if dev.type != "cuda":
            raise RuntimeError(f"FEARTracker (H100) needs a CUDA device, got {self.cuda_id!r}: there is no CPU path")
        return torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())

    def _preprocess_image(self, image: np.ndarray, transform=None) -> torch.Tensor:
        """uint8 HWC crop -> network input on the tracker's device.

        Default: upload the raw uint8 crop (1,H,W,3) -- 4x fewer bytes over PCIe -- and let the stem kernel
        apply the ImageNet normalisation with the reference's float32 roundings (bit-identical).  With
        ``host_normalize=True`` in the tracking config the crop is normalised on the host exactly like the
        reference (albumentations.Normalize + HWC->CHW) and uploaded as float32 (1,3,H,W)."""
        if self.tracking_config.get("host_normalize", False):
            chw = np.ascontiguousarray(np.transpose(image_ops.normalize(image[:, :, :3]), (2, 0, 1))[None])
            return torch.from_numpy(chw).pin_memory().to(self._device(), non_blocking=True)
        hwc = np.ascontiguousarray(image[:, :, :3][None])
        return torch.from_numpy(hwc).pin_memory().to(self._device(), non_blocking=True)

    def _rescale_bbox(self, bbox, padded_box):
        return image_ops.rescale_bbox(bbox, padded_box, self.tracking_config["instance_size"])

    def reset(self) -> None:
        self._template_features = None

    def initialize(self, image: np.ndarray, rect: np.ndarray, **kwargs) -> None:
        pass

    def update(self, image: np.ndarray, *kw) -> Dict[str, Any]:
        return {"bbox": self.tracking_state.bbox}


class FEARTracker(Tracker):
    def get_box_coder(self, tracking_config, cuda_id: int = 0):
        return FEARBoxCoder(tracker_config=tracking_config)

    def initialize(self, image: np.ndarray, rect: np.ndarray, **kwargs) -> None:
        """image: RGB uint8 HxWx3; rect: [x, y, w, h], 0-based."""
        rect = image_ops.clamp_bbox(rect, image.shape)
        st = self.tracking_state
        st.bbox = rect
        st.paths = deque([rect], maxlen=10)
        st.mean_color = np.mean(image, axis=(0, 1))
        self._template_features = self.get_template_features(image, rect)

    def get_template_features(self, image: np.ndarray, rect: np.ndarray) -> torch.Tensor:
        crop, _, _ = image_ops.extended_crop(image, rect, self.tracking_config["template_size"],
                                             self.tracking_config["template_bbox_offset"])
        return self.net.get_features(self._preprocess_image(crop))

    def update(self, image: np.ndarray, *kw) -> Dict[str, Any]:
        st, cfg = self.tracking_state, self.tracking_config
        if cfg.get("gpu_crop", False):
            return self._update_gpu_crop(image)
        crop, search_bbox, context = image_ops.extended_crop(image, st.bbox, cfg["instance_size"],
                                                             cfg["search_context"], st.mean_color)
        st.mapping = context
        st.prev_size = search_bbox[2:]
        pred_bbox, _ = self.track(crop)
        pred_bbox = image_ops.clamp_bbox(self._rescale_bbox(pred_bbox, context), image.shape)
        st.bbox = pred_bbox
        st.paths.append(pred_bbox)
        return dict(bbox=pred_bbox)

    def _update_gpu_crop(self, image: np.ndarray) -> Dict[str, Any]:
        """``gpu_crop=True``: the frame is uploaded once and the context crop + constant padding + bilinear resize of
        get_extended_crop (reference utils/utils.py:215-253) runs on the device (fear_crop_resize_u8, bit-identical
        to cv2's 8-bit fixed-point INTER_LINEAR) in the same CUDA graph as the network and the decode; the host only
        computes the integer context box and the 2 x 256 resize coefficients.  With ``smooth: true`` the network
        writes its maps and fear_decode_smooth runs the penalty, window and size smoothing of _smooth_postprocess in
        the same graph."""
        st, cfg = self.tracking_state, self.tracking_config
        if cfg.get("host_normalize", False) or image.shape[2] != 3:
            raise NotImplementedError("gpu_crop covers the default uint8 RGB tracking path (no smooth / host_normalize)")
        params, search_bbox, context = image_ops.crop_params(st.bbox, cfg["instance_size"], cfg["search_context"],
                                                             st.mean_color)
        st.mapping = context
        st.prev_size = search_bbox[2:]
        rec = self._track_record_gpu_crop(image, params)
        pred_bbox = np.array([rec["x"], rec["y"], rec["w"], rec["h"]])
        pred_bbox = image_ops.clamp_bbox(self._rescale_bbox(pred_bbox, context), image.shape)
        st.bbox = pred_bbox
        st.paths.append(pred_bbox)
        return dict(bbox=pred_bbox)

    def _track_record_gpu_crop(self, image: np.ndarray, params: np.ndarray):
        from . import _lib

        dev = self._device()
        size = int(self.tracking_config["instance_size"])
        h, w = image.shape[:2]
        cfg = self.tracking_config
        smooth = bool(cfg.get("smooth", False))
        st = getattr(self, "_gpu_crop_state", None)
        if st is None or st["device"] != dev or st["shape"] != (h, w) or st["params_pin"].numel() != params.size \
                or st["smooth"] != smooth:
            st = dict(device=dev, shape=(h, w), smooth=smooth,
                      frame_pin=torch.empty((h, w, 3), dtype=torch.uint8).pin_memory(),
                      frame=torch.empty((h, w, 3), dtype=torch.uint8, device=dev),
                      params_pin=torch.empty(params.size, dtype=torch.int32).pin_memory(),
                      params=torch.empty(params.size, dtype=torch.int32, device=dev),
                      crop=torch.empty((1, size, size, 3), dtype=torch.uint8, device=dev),
                      zf=torch.empty((1, 256, 8, 8), dtype=torch.float32, device=dev),
                      box_pin=torch.empty((1, 48), dtype=torch.uint8).pin_memory(),
                      graph=None, boxes=None, generation=None, zf_src=None, calls=0, graph_ok=True)
            if smooth:
                # fear_decode_smooth's inputs in one float64 buffer: prev_size (w, h), then its 259 params (penalty_k,
                # window_influence, lr, window).  The five scalars are copied per update, the window once here.
                st["smooth_pin"] = torch.empty(5, dtype=torch.float64).pin_memory()
                st["smooth_in"] = torch.empty(5 + 256, dtype=torch.float64, device=dev)
                st["smooth_in"][5:].copy_(torch.from_numpy(np.asarray(self.window, dtype=np.float64).reshape(256)))
                st["smooth_boxes"] = torch.empty((1, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8, device=dev)
            self._gpu_crop_state = st
        np.copyto(st["frame_pin"].numpy(), image)
        np.copyto(st["params_pin"].numpy(), params)
        st["frame"].copy_(st["frame_pin"], non_blocking=True)
        st["params"].copy_(st["params_pin"], non_blocking=True)
        if smooth:
            pw, ph = self.tracking_state.prev_size
            st["smooth_pin"].numpy()[:] = (pw, ph, cfg["penalty_k"], cfg["window_influence"], cfg["lr"])
            st["smooth_in"][:5].copy_(st["smooth_pin"], non_blocking=True)
        if st["zf_src"] is not self._template_features:
            st["zf"].copy_(self._template_features)
            st["zf_src"] = self._template_features
        lib = _lib.load()

        def step():
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(lib.fear_crop_resize_u8(st["frame"].data_ptr(), h, w, st["params"].data_ptr(), st["crop"].data_ptr(),
                                               size, stream), "fear_crop_resize_u8")
            if not smooth:
                return self.net.track_boxes(st["crop"], st["zf"])
            maps = self.net.track(st["crop"], st["zf"])  # maps only: the plain decode is skipped
            sp = st["smooth_in"].data_ptr()
            _lib.check(lib.fear_decode_smooth(maps[TARGET_REGRESSION_LABEL_KEY].data_ptr(),
                                              maps[TARGET_CLASSIFICATION_KEY].data_ptr(), 1, sp, sp + 16,
                                              st["smooth_boxes"].data_ptr(), stream), "fear_decode_smooth")
            return st["smooth_boxes"]

        use_graph = self.tracking_config.get("cuda_graph", True) and st["graph_ok"]
        if st["graph"] is not None and st["generation"] != self.net.generation():
            st["graph"], st["calls"] = None, 0  # stale pointers (see _track_record)
        if use_graph and st["graph"] is None and st["calls"] >= 1:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    st["boxes"] = step()
                st["graph"], st["generation"] = g, self.net.generation()
            except RuntimeError as exc:
                import warnings

                warnings.warn(f"FEARTracker: CUDA-graph capture of the gpu_crop step failed ({exc}); using eager launches")
                st["graph_ok"] = False
                torch.cuda.synchronize(dev)
        if use_graph and st["graph"] is not None and st["graph_ok"]:
            st["graph"].replay()
            boxes = st["boxes"]
        else:
            boxes = step()
        st["calls"] += 1
        st["box_pin"].copy_(boxes, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        return st["box_pin"].numpy().view(_lib.BOX_DTYPE).reshape(-1)[0].copy()

    def track(self, search_crop: np.ndarray) -> Tuple[np.ndarray, float]:
        if self.tracking_config.get("smooth", False):
            return self._postprocess(self.net.track(self._preprocess_image(search_crop), self._template_features))
        rec = self._track_record(search_crop)
        return np.array([rec["x"], rec["y"], rec["w"], rec["h"]]), np.float32(rec["score"])

    # -- streaming fast path: persistent pinned staging + (optionally) the whole per-frame step as ONE CUDA graph --
    def _track_record(self, search_crop: np.ndarray):
        """One frame: crop -> pinned staging -> device -> network + on-device decode -> 48-byte box record.

        The 70 kernel launches of a batch-1 step cost more host time than GPU time, so after one eager warm-up
        call the step is captured into a CUDA graph (static input / template / output buffers; the library's
        workspace pointers are stable) and replayed per frame.  ``cuda_graph=False`` in the tracking config keeps
        eager launches."""
        dev = self._device()
        st = getattr(self, "_stream_state", None)
        host_norm = bool(self.tracking_config.get("host_normalize", False))
        if st is None or st["device"] != dev or st["host_norm"] != host_norm:
            shape, dtype = ((1, 3, 256, 256), torch.float32) if host_norm else ((1, 256, 256, 3), torch.uint8)
            st = dict(device=dev, host_norm=host_norm, pin=torch.empty(shape, dtype=dtype).pin_memory(),
                      dev=torch.empty(shape, dtype=dtype, device=dev),
                      zf=torch.empty((1, 256, 8, 8), dtype=torch.float32, device=dev),
                      box_pin=torch.empty((1, 48), dtype=torch.uint8).pin_memory(),
                      graph=None, boxes=None, generation=None, zf_src=None, calls=0, graph_ok=True)
            self._stream_state = st
        if host_norm:
            np.copyto(st["pin"].numpy(), np.transpose(image_ops.normalize(search_crop[:, :, :3]), (2, 0, 1))[None])
        else:
            np.copyto(st["pin"].numpy(), search_crop[None, :, :, :3])
        st["dev"].copy_(st["pin"], non_blocking=True)
        if st["zf_src"] is not self._template_features:  # new template (initialize / reset): refresh the static copy
            st["zf"].copy_(self._template_features)
            st["zf_src"] = self._template_features
        use_graph = self.tracking_config.get("cuda_graph", True) and st["graph_ok"]
        if st["graph"] is not None and st["generation"] != self.net.generation():
            # weights re-packed, workspace re-allocated by a larger batch on the same net, or an option changed:
            # the pointers / kernels baked into the captured graph are stale -> warm up eagerly and capture again
            st["graph"], st["calls"] = None, 0
        if use_graph and st["graph"] is None and st["calls"] >= 1:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    st["boxes"] = self.net.track_boxes(st["dev"], st["zf"])
                st["graph"], st["generation"] = g, self.net.generation()
            except RuntimeError as exc:  # capture failed: stay eager for this tracker, loudly
                import warnings

                warnings.warn(f"FEARTracker: CUDA-graph capture of the per-frame step failed ({exc}); "
                              "falling back to eager launches (slower streaming path)")
                st["graph_ok"] = False
                torch.cuda.synchronize(dev)
        if use_graph and st["graph"] is not None and st["graph_ok"]:
            st["graph"].replay()
            boxes = st["boxes"]
        else:
            boxes = self.net.track_boxes(st["dev"], st["zf"])
        st["calls"] += 1
        st["box_pin"].copy_(boxes, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        from . import _lib

        return st["box_pin"].numpy().view(_lib.BOX_DTYPE).reshape(-1)[0].copy()

    # -- reference-shaped post-processing on a maps dictionary (used for the optional smoothing) --
    def _postprocess(self, track_result: Dict[str, torch.Tensor]) -> Tuple[np.ndarray, float]:
        reg = track_result[TARGET_REGRESSION_LABEL_KEY].detach().float()
        cls_score = track_result[TARGET_CLASSIFICATION_KEY].detach().float().sigmoid()
        if not self.tracking_config.get("smooth", False):
            rec = self.box_coder.decode_records(reg, cls_score, use_sigmoid=False)[0]
            return np.array([rec["x"], rec["y"], rec["w"], rec["h"]]), np.float32(rec["score"])
        return self._smooth_postprocess(reg.cpu().numpy()[0].astype(np.float64), cls_score.cpu().numpy()[0, 0])

    def _smooth_postprocess(self, reg: np.ndarray, score: np.ndarray) -> Tuple[np.ndarray, float]:
        """Scale/ratio penalty + cosine window + size smoothing (reference base_tracker.py:126-205),
        256-element float64 host math; only active when the config carries ``smooth: true``."""
        cfg, st = self.tracking_config, self.tracking_state
        gx, gy = self.box_coder.grid_x.cpu().numpy()[0], self.box_coder.grid_y.cpu().numpy()[0]
        x1, y1, x2, y2 = gx - reg[0], gy - reg[1], gx + reg[2], gy + reg[3]

        def limit(r):
            return np.maximum(r, 1.0 / r)

        def sq(w, h):
            pad = (w + h) * 0.5
            return np.sqrt((w + pad) * (h + pad))

        pw, ph = st.prev_size
        s_c = limit(sq(x2 - x1, y2 - y1) / sq(pw, ph))
        r_c = limit((pw / ph) / ((x2 - x1) / (y2 - y1)))
        penalty = np.exp(-(r_c * s_c - 1) * cfg["penalty_k"])
        pscore = penalty * score
        pscore = pscore * (1 - cfg["window_influence"]) + self.window * cfg["window_influence"]
        flat = int(np.argmax(pscore))
        r, c = flat // 16, flat % 16
        box = np.array([x1[r, c], y1[r, c], x2[r, c] - x1[r, c], y2[r, c] - y1[r, c]])
        # the reference multiplies a float64 numpy scalar into a float32 torch scalar (base_tracker.py:158): the size
        # learning rate is therefore rounded to float32 at each step -- reproduced here so boxes match to the last bit
        lr = (float(penalty[r, c]) * torch.tensor(score[r, c], dtype=torch.float32) * cfg["lr"]).item()
        size, prev = box[2:] * lr, np.asarray(st.prev_size) * (1 - lr)
        w = prev[0] + lr * (size[0] + prev[0])
        h = prev[1] + lr * (size[1] + prev[1])
        return np.array([box[0], box[1], w, h]), score[r, c]
