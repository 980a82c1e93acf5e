"""FEARTracker: stateful single-object tracker around the H100 FEARNet.

API mirror of reference model_training/tracker/base_tracker.py:28-124 and fear_tracker.py:13-86:
``FEARTracker(model, cuda_id=0, **tracking_config)``, ``initialize(image, rect)``,
``update(image) -> {"bbox": [x, y, w, h]}``, ``track(search_crop)``, ``get_template_features``,
``to_device``, ``reset``.  Cropping / normalisation stay on the host (cv2 fixed-point resize is part
of the reference's observable behaviour); network + decode run in libfear_b200 and only the
48-byte box record comes back per frame.  With ``gpu_crop: true`` the numpy frame is uploaded and cropped on the device.

Frames already in GPU memory -- uint8 (H, W, 3) CUDA tensors with any non-negative strides, YUV420Frame /
YUV422Frame / YUV444Frame decoder surfaces, V210Frame capture buffers, BayerFrame raw mosaics, MonoFrame
single-channel frames and RGBFrame BGR / BGRA / ABGR, 10-bit, 16-bit and planar RGB frames -- are read in place:
the crop, the conversion to RGB (or the demosaic), the network and the decode (plain or smoothed) run on the device, and
the tracker returns exactly what it returns for the same pixels as a numpy array (``image_ops.yuv_to_rgb`` of a YUV
frame's planes, ``image_ops.bayer_to_rgb`` of a Bayer frame's codes, ``image_ops.mono_to_rgb`` of a mono frame's,
``image_ops.rgb_frame_to_rgb`` of an RGB frame's samples).  Any of them may be wrapped in ``Oriented(frame, rotate,
mirror)`` (phone video's display rotation, a camera mounted upside down or mirrored): the tracker then sees
``image_ops.orient`` of that frame, oriented inside the crop.
"""
from collections import deque
from typing import Any, Dict, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn as nn

from . import image_ops, multi_tracker
from .box_coder import FEARBoxCoder, TrackerDecodeResult
from .constants import TARGET_CLASSIFICATION_KEY, TARGET_REGRESSION_LABEL_KEY


# byte layout of FEARTracker's device-frame inputs: the frame's table record (up to a FearFrameYCbCrHDR; a
# FearFrameBayer is 40 bytes, a FearFrameMono 48, a FearFrameRGB 72), the int32 orientation code of an Oriented frame
# (8 bytes kept), a FearTarget, then five float64 inputs of fear_decode_smooth, which the window follows on the device
_ORIENT_OFFSET = 104
_TARGET_OFFSET = _ORIENT_OFFSET + 8
_SMOOTH_OFFSET = _TARGET_OFFSET + 64
_DEVICE_INPUT_BYTES = _SMOOTH_OFFSET + 5 * 8


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
    """The reference's single-object tracker.  ``initialize``, ``update`` and ``get_template_features`` take a frame as
    a uint8 (H, W, 3) RGB numpy array, as a uint8 (H, W, 3) CUDA tensor on the tracker's device (any non-negative
    strides: ``rgba[..., :3]``, ``chw.permute(1, 2, 0)``, a region of interest), or as a YUV420Frame, YUV422Frame,
    YUV444Frame, V210Frame, BayerFrame, MonoFrame or RGBFrame whose planes, words or samples are on the tracker's
    device; the kind may change from one call to the next.

    Numpy frames take the host crop, or with ``gpu_crop: true`` an upload and the device crop.  Device frames always
    take the device step, whatever ``gpu_crop`` says, since the host crop could only read them after copying them back:
    fear_crop_targets_view_u8 (tensors), fear_crop_targets_ycbcr_u8 (YUV frames, converted to RGB inside the crop),
    fear_crop_targets_ycbcr_v210_u8 (v210 frames, unpacked and converted inside the crop), fear_crop_targets_bayer_u8
    (Bayer frames, demosaiced inside the crop), fear_crop_targets_mono_u8 (mono frames, mapped to grey inside the
    crop, after fear_frame_range_mono when the frame has gain control) or fear_crop_targets_rgb_u8 (RGB frames in any
    channel order and container, mapped to 8 bits inside the crop) makes the search crop, then the network and the
    decode, plain or with ``smooth: true`` the smoothed one, run as one CUDA graph and one 48-byte record comes back.
    The results, ``tracking_state`` included, are those of the same tracker fed the same pixels as numpy arrays
    (``image_ops.yuv_to_rgb`` of a YUV frame's planes with its ``CHROMA_SHIFT``, of a v210 frame's
    ``image_ops.v210_unpack`` planes, ``image_ops.bayer_to_rgb`` of a Bayer frame's codes, ``image_ops.mono_to_rgb``
    of a mono frame's codes with its ``agc``, ``image_ops.rgb_frame_to_rgb`` of an RGB frame's samples).  An
    ``Oriented`` device frame takes the table's oriented crop (fear_crop_targets_oriented_u8) with its code staged in
    the same input copy, and gives what ``image_ops.orient`` of the frame it wraps gives as a numpy array; rects and
    boxes are in the turned picture's coordinates.  Device frames must be ready on the current CUDA stream; every call
    synchronises it before it returns, so they only need to live for the call.
    ``host_normalize: true`` takes numpy frames only."""

    def get_box_coder(self, tracking_config, cuda_id: int = 0):
        size, stride, score = (tracking_config[k] for k in ("instance_size", "total_stride", "score_size"))
        if isinstance(stride, int) and stride > 0 and score != size // stride:
            raise ValueError(f"score_size must be instance_size // total_stride = {size // stride}, got {score}")
        return FEARBoxCoder(tracker_config=tracking_config)

    def _score_cells(self) -> int:
        return int(self.tracking_config["score_size"]) ** 2

    def initialize(self, image: np.ndarray, rect: np.ndarray, **kwargs) -> None:
        """image: RGB uint8 HxWx3 (or a device frame, see the class docstring); rect: [x, y, w, h], 0-based."""
        kind = self._frame_kind(image)
        rect = image_ops.clamp_bbox(rect, image.shape)
        st = self.tracking_state
        if kind != "numpy":
            mean_color = self._device_mean_color(image, kind)
            features = self._device_template_features(image, kind, rect, mean_color)
            st.bbox, st.paths, st.mean_color = rect, deque([rect], maxlen=10), mean_color
            self._template_features = features
            return
        st.bbox = rect
        st.paths = deque([rect], maxlen=10)
        st.mean_color = np.mean(image, axis=(0, 1))
        self._template_features = self.get_template_features(image, rect)

    def get_template_features(self, image: np.ndarray, rect: np.ndarray) -> torch.Tensor:
        kind = self._frame_kind(image)
        if kind != "numpy":
            return self._device_template_features(image, kind, rect, self._device_mean_color(image, kind))
        crop, _, _ = image_ops.extended_crop(image, rect, self.tracking_config["template_size"],
                                             self.tracking_config["template_bbox_offset"])
        return self.net.get_features(self._preprocess_image(crop))

    def update(self, image: np.ndarray, *kw) -> Dict[str, Any]:
        st, cfg = self.tracking_state, self.tracking_config
        kind = self._frame_kind(image)
        if kind != "numpy":
            return self._update_device_frame(image, kind)
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
        computes the integer context box and the 2 x instance_size resize coefficients.  With ``smooth: true`` the
        network writes its maps and fear_decode_smooth_sized runs the penalty, window and size smoothing of
        _smooth_postprocess in the same graph."""
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
                # fear_decode_smooth_sized's inputs in one float64 buffer: prev_size (w, h), then its 3 + s * s params
                # (penalty_k, window_influence, lr, window).  The five scalars are copied per update, the window once here.
                cells = self._score_cells()
                st["smooth_pin"] = torch.empty(5, dtype=torch.float64).pin_memory()
                st["smooth_in"] = torch.empty(5 + cells, dtype=torch.float64, device=dev)
                st["smooth_in"][5:].copy_(torch.from_numpy(np.asarray(self.window, dtype=np.float64).reshape(cells)))
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
            _lib.check(lib.fear_decode_smooth_sized(maps[TARGET_REGRESSION_LABEL_KEY].data_ptr(),
                                                    maps[TARGET_CLASSIFICATION_KEY].data_ptr(), 1, size // 16, sp,
                                                    sp + 16, st["smooth_boxes"].data_ptr(), stream),
                       "fear_decode_smooth_sized")
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

    # -- device frames: CUDA tensors and YUV frames, read in place by the crop-targets entry points (one target) --
    def _frame_kind(self, image) -> str:
        """"numpy", "cuda", "yuv", "bayer", "mono" or "rgb" (multi_tracker.frame_kind).  A device frame is checked here, before
        any device call or state change: NotImplementedError with ``host_normalize``, ValueError when malformed."""
        kind = multi_tracker.frame_kind(image)
        if kind == "numpy":
            return kind
        if self.tracking_config.get("host_normalize", False):
            raise NotImplementedError("host_normalize normalises numpy crops on the host; device frames (CUDA tensors, "
                                      "YUV frames) are normalised on the device: drop host_normalize to track on them")
        multi_tracker.check_device_frame(0, image, kind, self._device)
        return kind

    def _device_frame_state(self) -> dict:
        """Buffers of the device-frame step, separate from the gpu_crop path's.  ``inputs`` (pinned) and ``dev_in``
        share one layout, sent with one host-to-device copy per call: the frame's table record (a FearFrameView, a
        FearFrameYCbCr, a FearFrameYCbCrV210, a FearFrameYCbCrHDR, a FearFrameBayer, a FearFrameMono or a FearFrameRGB)
        at byte 0, an Oriented frame's int32 code at byte 104, the FearTarget at byte 112, fear_decode_smooth's
        prev_size (w, h), penalty_k, window_influence and lr as float64 at byte 176; then, on the device only, the
        score_size x score_size window."""
        from . import _lib

        dev = self._device()
        smooth = bool(self.tracking_config.get("smooth", False))
        st = getattr(self, "_device_state", None)
        if st is not None and st["device"] == dev and st["smooth"] == smooth:
            return st
        size, tsize = int(self.tracking_config["instance_size"]), int(self.tracking_config["template_size"])
        st = dict(device=dev, smooth=smooth,
                  inputs=torch.zeros(_DEVICE_INPUT_BYTES, dtype=torch.uint8).pin_memory(),
                  dev_in=torch.zeros(_DEVICE_INPUT_BYTES + self._score_cells() * 8, dtype=torch.uint8, device=dev),
                  crop=torch.empty((1, size, size, 3), dtype=torch.uint8, device=dev),
                  tcrop=torch.empty((1, tsize, tsize, 3), dtype=torch.uint8, device=dev),
                  sums=torch.empty((1, 3), dtype=torch.int64, device=dev),
                  sums_pin=torch.empty((1, 3), dtype=torch.int64).pin_memory(),
                  zf=torch.empty((1, 256, 8, 8), dtype=torch.float32, device=dev),
                  smooth_boxes=torch.empty((1, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8, device=dev),
                  box_pin=torch.empty((1, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8).pin_memory(),
                  graph=None, boxes=None, key=None, zf_src=None, calls=0, graph_ok=True)
        window = np.asarray(self.window, dtype=np.float64).reshape(self._score_cells())
        st["dev_in"][_DEVICE_INPUT_BYTES:].copy_(torch.from_numpy(window).view(torch.uint8))
        self._device_state = st
        return st

    def _stage_device_inputs(self, st: dict, image, kind: str, bbox, pad, prev_size=None) -> str:
        """Write the frame's record, the target (frame 0, ``bbox``, padding colour ``pad``) and, given ``prev_size``,
        the smooth scalars into the pinned inputs and send them with one host-to-device copy.  Returns the table name:
        "views" for a tensor, "ycbcr_hdr" for a YUV frame with a transfer (PQ, HLG), "ycbcr_v210" for another
        V210Frame, "ycbcr" for every other YUV frame, "bayer" for a BayerFrame, "mono" for a MonoFrame, "rgb" for an
        RGBFrame."""
        frame = multi_tracker.stored(image)
        table = kind if kind in ("bayer", "mono", "rgb") else "views"
        if kind == "yuv":
            table = "ycbcr_v210" if isinstance(frame, multi_tracker.V210Frame) else "ycbcr"
            if frame.transfer is not None:
                table = "ycbcr_hdr"
        raw, dtype = st["inputs"].numpy(), multi_tracker.TABLE_DTYPES[table]
        multi_tracker.write_records(raw[:dtype.itemsize].view(dtype), [image], table)
        target = raw[_TARGET_OFFSET:_SMOOTH_OFFSET].view(np.int32)
        target[:] = 0
        target[1:5] = bbox
        target[9:12] = pad
        if prev_size is not None:
            cfg = self.tracking_config
            raw[_SMOOTH_OFFSET:].view(np.float64)[:] = (prev_size[0], prev_size[1], cfg["penalty_k"],
                                                        cfg["window_influence"], cfg["lr"])
        if isinstance(image, multi_tracker.Oriented):
            raw[_ORIENT_OFFSET:_ORIENT_OFFSET + 4].view(np.int32)[0] = image.code
        st["dev_in"][:_DEVICE_INPUT_BYTES].copy_(st["inputs"], non_blocking=True)
        return table

    @staticmethod
    def _device_frame_range(st: dict, image, kind: str, stream) -> None:
        """For a MonoFrame with gain control, fear_frame_range_mono on the staged FearFrameMono record: the frame's code
        range, which the mono sums and crop read, written into the record on the device."""
        from . import _lib

        if multi_tracker.uses_agc([image], kind):
            fn = multi_tracker.RANGE_ENTRY_POINT
            _lib.check(getattr(_lib.load(), fn)(st["dev_in"].data_ptr(), 1, stream), fn)

    @staticmethod
    def _device_crop(st: dict, image, table: str, offset: float, size: int, out_ptr: int, stream) -> None:
        """The crop-targets entry point of ``table`` on the staged record and FearTarget (one frame, one target), or
        for an ``Oriented`` frame the oriented one reading the staged code."""
        from . import _lib

        lib, dp = _lib.load(), st["dev_in"].data_ptr()
        if isinstance(image, multi_tracker.Oriented):
            fn = multi_tracker.ORIENTED_ENTRY_POINTS[0]
            _lib.check(getattr(lib, fn)(_lib.ORIENT_TABLES[table], dp, dp + _ORIENT_OFFSET, 1, dp + _TARGET_OFFSET, 1,
                                        offset, size, out_ptr, stream), fn)
        else:
            fn = multi_tracker.ENTRY_POINTS[table][1]
            _lib.check(getattr(lib, fn)(dp, 1, dp + _TARGET_OFFSET, 1, offset, size, out_ptr, stream), fn)

    def _device_mean_color(self, image, kind: str) -> np.ndarray:
        """np.mean(frame, axis=(0, 1)) of the RGB frame, bit for bit: exact per-channel sums on the device over H * W."""
        from . import _lib

        st = self._device_frame_state()
        dev = st["device"]
        with torch.cuda.device(dev):
            table = self._stage_device_inputs(st, image, kind, (0, 0, 0, 0), (0, 0, 0))
            sums_fn = multi_tracker.ENTRY_POINTS[table][0]
            stream = torch.cuda.current_stream(dev)
            self._device_frame_range(st, image, kind, stream.cuda_stream)
            _lib.check(getattr(_lib.load(), sums_fn)(st["dev_in"].data_ptr(), 1, st["sums"].data_ptr(),
                                                     stream.cuda_stream), sums_fn)
            st["sums_pin"].copy_(st["sums"], non_blocking=True)
            stream.synchronize()
        h, w = image.shape[:2]
        return st["sums_pin"].numpy()[0].view(np.uint64).astype(np.float64) / (h * w)

    def _device_template_features(self, image, kind: str, rect, mean_color) -> torch.Tensor:
        """The template of get_template_features: the 128 x 128 context crop (offset template_bbox_offset) made by the
        crop-targets entry point on a one-row FearTarget, then net.get_features on the uint8 crop."""
        from . import _lib

        cfg = self.tracking_config
        size, offset = int(cfg["template_size"]), float(cfg["template_bbox_offset"])
        box = np.asarray(rect, dtype=np.float64)
        if box.shape != (4,) or not np.array_equal(box, np.trunc(box)) or np.abs(box).max() > 2 ** 31 - 1:
            raise ValueError(f"a device frame's template box must be 4 integers [x, y, w, h], got {rect!r}")
        image_ops.crop_geometry(box, size, offset)  # the IndexError of a zero-area box, as extended_crop raises it
        st = self._device_frame_state()
        dev = st["device"]
        with torch.cuda.device(dev):
            table = self._stage_device_inputs(st, image, kind, box.astype(np.int32), image_ops.padding_color(mean_color))
            stream = torch.cuda.current_stream(dev)
            self._device_frame_range(st, image, kind, stream.cuda_stream)
            self._device_crop(st, image, table, offset, size, st["tcrop"].data_ptr(), stream.cuda_stream)
            features = self.net.get_features(st["tcrop"])
            stream.synchronize()  # the pinned inputs are rewritten by the next call
        return features

    def _update_device_frame(self, image, kind: str) -> Dict[str, Any]:
        st, cfg = self.tracking_state, self.tracking_config
        search_bbox, context = image_ops.crop_geometry(st.bbox, cfg["instance_size"], cfg["search_context"])
        st.mapping = context
        st.prev_size = search_bbox[2:]
        rec = self._track_record_device_frame(image, kind)
        pred_bbox = np.array([rec["x"], rec["y"], rec["w"], rec["h"]])
        pred_bbox = image_ops.clamp_bbox(self._rescale_bbox(pred_bbox, context), image.shape)
        st.bbox = pred_bbox
        st.paths.append(pred_bbox)
        return dict(bbox=pred_bbox)

    def _track_record_device_frame(self, image, kind: str):
        """One update on a device frame: crop-targets (N = 1, search_context, instance_size) -> fear_track_sized_u8 -> the
        plain decode, or with smooth the maps -> fear_decode_smooth_sized; one 48-byte record back.  The crop kernel reads the frame's record
        when it runs, so the graph (captured on the second update) keys on the table kind, smooth, the input buffer,
        whether it starts with the mono range kernel, whether the frame is ``Oriented`` and net.generation(), not on the
        frame's address, shape or orientation code: fresh decoder surfaces, a resolution change and a new rotation
        replay it."""
        from . import _lib

        st = self._device_frame_state()
        dev, smooth, cfg = st["device"], st["smooth"], self.tracking_config
        size = int(cfg["instance_size"])
        with torch.cuda.device(dev):
            trk = self.tracking_state
            table = self._stage_device_inputs(st, image, kind, trk.bbox, image_ops.padding_color(trk.mean_color),
                                              trk.prev_size if smooth else None)
            if st["zf_src"] is not self._template_features:
                st["zf"].copy_(self._template_features)
                st["zf_src"] = self._template_features
            lib = _lib.load()
            agc = multi_tracker.uses_agc([image], kind)
            oriented = isinstance(image, multi_tracker.Oriented)

            def step():
                stream = torch.cuda.current_stream(dev).cuda_stream
                self._device_frame_range(st, image, kind, stream)
                dp = st["dev_in"].data_ptr()
                self._device_crop(st, image, table, float(cfg["search_context"]), size, st["crop"].data_ptr(), stream)
                if not smooth:
                    return self.net.track_boxes(st["crop"], st["zf"])
                maps = self.net.track(st["crop"], st["zf"])
                sp = dp + _SMOOTH_OFFSET
                _lib.check(lib.fear_decode_smooth_sized(maps[TARGET_REGRESSION_LABEL_KEY].data_ptr(),
                                                        maps[TARGET_CLASSIFICATION_KEY].data_ptr(), 1, size // 16, sp,
                                                        sp + 16, st["smooth_boxes"].data_ptr(), stream),
                           "fear_decode_smooth_sized")
                return st["smooth_boxes"]

            key = (table, smooth, st["dev_in"].data_ptr(), self.net.generation(), agc, oriented)
            if key != st["key"]:  # another entry point, or stale workspace / weight pointers: warm up and capture again
                st["graph"], st["key"], st["calls"] = None, key, 0
            use_graph = cfg.get("cuda_graph", True) and st["graph_ok"]
            if use_graph and st["graph"] is None and st["calls"] >= 1:
                try:
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        st["boxes"] = step()
                    st["graph"] = g
                except RuntimeError as exc:
                    import warnings

                    warnings.warn(f"FEARTracker: CUDA-graph capture of the device-frame step failed ({exc}); "
                                  "using eager launches")
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
            size = int(self.tracking_config["instance_size"])
            shape, dtype = ((1, 3, size, size), torch.float32) if host_norm else ((1, size, size, 3), torch.uint8)
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
        score_size x score_size float64 host math; only active when the config carries ``smooth: true``."""
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
        r, c = divmod(flat, pscore.shape[1])
        box = np.array([x1[r, c], y1[r, c], x2[r, c] - x1[r, c], y2[r, c] - y1[r, c]])
        # the reference multiplies a float64 numpy scalar into a float32 torch scalar (base_tracker.py:158): the size
        # learning rate is therefore rounded to float32 at each step -- reproduced here so boxes match to the last bit
        lr = (float(penalty[r, c]) * torch.tensor(score[r, c], dtype=torch.float32) * cfg["lr"]).item()
        size, prev = box[2:] * lr, np.asarray(st.prev_size) * (1 - lr)
        w = prev[0] + lr * (size[0] + prev[0])
        h = prev[1] + lr * (size[1] + prev[1])
        return np.array([box[0], box[1], w, h]), score[r, c]
