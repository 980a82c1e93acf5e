"""FEARMultiTracker: many targets, in one or several video streams, stepped together once per frame.

    trk = FEARMultiTracker(net, cuda_id=0, max_targets=64, **FEAR_XS_TRACKER_KWARGS)
    ids = trk.add(frames, rects, streams=None)   # frames: one HxWx3 uint8 array or a list of F; streams -> frame index
    out = trk.update(frames)                      # {"bbox": (N,4) int64, "score": (N,) float32, "ids": (N,) int64}
    trk.remove(ids); trk.reset()

Frames are numpy arrays in host memory or uint8 (H, W, 3) CUDA tensors already on the tracker's device, strided views
included (t[..., :3] of an RGBA surface, t.permute(1, 2, 0) of a CHW tensor, t[y0:y1, x0:x1]); tensors are read where
they are, without a copy.

Every target behaves exactly like its own ``FEARTracker(gpu_crop=True)`` started on the same frame with the same
rect: the rect is clamped, the padding colour is the mean colour of the init frame, the template is the network
features of its 128 x 128 context crop, and each frame runs crop -> network -> decode -> rescale -> clamp.  Instead of
one batch-1 step and one host round trip per target, one step runs all N targets at batch N:

    fear_crop_targets_view_u8 (N search crops)  ->  fear_track_u8 (B = N, Bz = N)  ->  fear_advance_targets_view

on per-target state kept in device memory (an (N, 16) int32 tensor of FearTarget records, include/fear_b200.h), so the
step is captured once as a CUDA graph and replayed every frame.  The kernels find the frames through a table of
FearFrameView records (address, byte strides, H, W) in a fixed device buffer, written before every step: numpy frames
are packed into one pinned buffer and sent with one copy, and their views point into the packed device buffer; CUDA
tensors' views point at the tensors.  The host then reads back the boxes and scores.  The launch count of a step
depends neither on N nor on the kind of frames.
"""
import math
import warnings
from typing import Any, Dict, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib, image_ops

_FRAME_ALIGN = 16  # byte alignment of each frame inside the packed buffer
_MAX_SIDE = 2 ** 31 - 1  # H and W are int32 in FearFrameView


def frame_view(frame: torch.Tensor) -> tuple:
    """The FearFrameView record (data, row_stride, pixel_stride, channel_stride, H, W) of a uint8 (H, W, 3) tensor, as
    it lies in memory: the address of pixel (0, 0) channel R and the byte strides (a uint8 stride is a byte stride)."""
    rs, ps, cs = frame.stride()
    return (frame.data_ptr(), rs, ps, cs, frame.shape[0], frame.shape[1])


class FEARMultiTracker:
    def __init__(self, model, cuda_id: Union[int, str] = 0, max_targets: int = 64, **tracking_config: Any) -> None:
        cfg = tracking_config
        if cfg.get("smooth", False) or cfg.get("host_normalize", False):
            raise NotImplementedError("FEARMultiTracker covers the default uint8 RGB tracking path "
                                      "(no smooth / host_normalize)")
        for key in ("search_context", "template_bbox_offset"):
            v = float(cfg[key])
            if not math.isfinite(v) or v < 0:
                raise ValueError(f"{key} must be finite and >= 0, got {cfg[key]!r}")
        if int(cfg["instance_size"]) != 256 or int(cfg["template_size"]) != 128:
            raise ValueError("FEAR-XS tracks 256 x 256 search crops against 128 x 128 templates; got instance_size="
                             f"{cfg['instance_size']}, template_size={cfg['template_size']}")
        if int(max_targets) < 1:
            raise ValueError(f"max_targets must be >= 1, got {max_targets}")
        self.net = model
        self.cuda_id = cuda_id
        self.tracking_config = tracking_config
        self.max_targets = int(max_targets)
        self.net.reserve(self.max_targets)  # the whole batch fits the workspace: graph capture never allocates
        self._buf = None  # device buffers, allocated on first use
        self._frames_key = None  # numpy frame shapes the packed buffer is laid out for
        self._graph = None
        self._graph_key = None
        self._graph_gen = None
        self._graph_ok = True
        self._calls = 0
        self.reset()

    # ------------------------------------------------------------------ public API
    def reset(self) -> None:
        """Drop every target (ids start again from 0)."""
        self._ids = np.zeros(0, dtype=np.int64)
        self._streams = np.zeros(0, dtype=np.int64)
        self._next_id = 0

    def initialize(self, frames, rects, streams: Optional[Sequence[int]] = None) -> np.ndarray:
        self.reset()
        return self.add(frames, rects, streams)

    @property
    def ids(self) -> np.ndarray:
        return self._ids.copy()

    def __len__(self) -> int:
        return len(self._ids)

    def add(self, frames, rects, streams: Optional[Sequence[int]] = None) -> np.ndarray:
        """Start tracking ``rects`` ((n, 4) [x, y, w, h]); target i lives in stream ``streams[i]`` (default 0), whose
        current frame is ``frames[streams[i]]``.  Returns the new targets' ids.

        ``frames`` are all numpy arrays or all CUDA tensors (see ``update``).  A target's padding colour is the mean
        colour of its frame, from exact per-channel sums computed on the device."""
        frames, on_device = self._check_frames(frames)
        rects = np.asarray(rects, dtype=np.float64)
        if rects.ndim == 1 and rects.size == 4:
            rects = rects[None]
        if rects.ndim != 2 or rects.shape[1] != 4:
            raise ValueError(f"rects must be (n, 4) [x, y, w, h], got shape {rects.shape}")
        n = rects.shape[0]
        streams = self._check_streams(np.zeros(n, dtype=np.int64) if streams is None else streams, n, len(frames))
        if len(self._ids) + n > self.max_targets:
            raise ValueError(f"{len(self._ids)} + {n} targets exceed max_targets = {self.max_targets}")
        if n == 0:
            return np.zeros(0, dtype=np.int64)
        cfg = self.tracking_config
        recs = np.zeros((n, _lib.TARGET_INTS), dtype=np.int32)
        for i, (rect, s) in enumerate(zip(rects, streams)):
            box = image_ops.clamp_bbox(rect, tuple(frames[s].shape))
            ctx = image_ops.context_box(box, cfg["template_bbox_offset"])
            inner = image_ops.trim_box([box[0] - ctx[0], box[1] - ctx[1], box[2], box[3]], (ctx[3], ctx[2]))
            if inner[2] * inner[3] == 0:
                raise IndexError("target box has zero area inside its context crop")
            recs[i, 0] = s
            recs[i, 1:5] = box
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            num_frames = len(frames)
            self._upload_frames(frames, on_device, dev)
            lib = _lib.load()
            stream = torch.cuda.current_stream(dev)
            _lib.check(lib.fear_frame_sums_u8(b["views"].data_ptr(), num_frames, b["sums"].data_ptr(),
                                              stream.cuda_stream), "fear_frame_sums_u8")
            b["sums_pin"][:num_frames].copy_(b["sums"][:num_frames], non_blocking=True)
            stream.synchronize()
            # numpy's mean of uint8 is an exact float64 sum of integers over H * W; then cv::saturate_cast, as
            # FEARTracker's padding
            sums = b["sums_pin"].numpy()[:num_frames].view(np.uint64)
            pixels = np.array([f.shape[0] * f.shape[1] for f in frames], dtype=np.float64)
            pads = np.clip(np.rint(sums / pixels[:, None]), 0, 255).astype(np.int32)
            recs[:, 9:12] = pads[streams]
            n0 = len(self._ids)
            b["state"][n0:n0 + n].copy_(torch.from_numpy(recs).pin_memory(), non_blocking=True)
            size = int(cfg["template_size"])
            crops = b["tcrops"][:n]
            _lib.check(lib.fear_crop_targets_view_u8(b["views"].data_ptr(), num_frames, b["state"][n0].data_ptr(), n,
                                                     float(cfg["template_bbox_offset"]), size, crops.data_ptr(),
                                                     stream.cuda_stream), "fear_crop_targets_view_u8")
            b["zf"][n0:n0 + n].copy_(self.net.get_features(crops))
            stream.synchronize()  # the pinned staging buffers are reused by the next call
        new_ids = np.arange(self._next_id, self._next_id + n, dtype=np.int64)
        self._next_id += n
        self._ids = np.concatenate([self._ids, new_ids])
        self._streams = np.concatenate([self._streams, streams])
        return new_ids

    def remove(self, ids) -> None:
        ids = np.atleast_1d(np.asarray(ids, dtype=np.int64))
        unknown = np.setdiff1d(ids, self._ids)
        if unknown.size:
            raise ValueError(f"unknown target ids {unknown.tolist()}")
        keep = np.flatnonzero(~np.isin(self._ids, ids))
        if self._buf is not None and keep.size:
            with torch.cuda.device(self._buf["device"]):
                idx = torch.from_numpy(keep).to(self._buf["device"])
                m = keep.size
                self._buf["state"][:m] = self._buf["state"][idx]
                self._buf["zf"][:m] = self._buf["zf"][idx]
        self._ids, self._streams = self._ids[keep], self._streams[keep]

    def update(self, frames) -> Dict[str, np.ndarray]:
        """One frame of every stream -> the new box and score of every target, in the order of ``ids``.

        ``frames`` (one frame or a list of F, stream i's frame at index i) are either all ``np.ndarray`` or all
        ``torch.Tensor``; the kind may change from one call to the next.  A tensor frame is uint8 of shape (H, W, 3)
        on the tracker's CUDA device, with any non-negative strides: views are read as they are, nothing is copied.
        Tensor frames must be ready on the current CUDA stream (write them on that stream, or make it wait for the
        stream that did, as for any torch op).  ``update`` synchronises that stream before it returns, so the tensors
        only need to live until the call returns."""
        frames, on_device = self._check_frames(frames)
        n = len(self._ids)
        if n and int(self._streams.max()) >= len(frames):
            raise ValueError(f"targets track stream {int(self._streams.max())} but only {len(frames)} frames were given")
        if n == 0:
            return dict(bbox=np.zeros((0, 4), dtype=np.int64), score=np.zeros(0, dtype=np.float32),
                        ids=self._ids.copy())
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            self._upload_frames(frames, on_device, dev)
            boxes = self._run_step(n, len(frames), dev)
            b["state_pin"][:n].copy_(b["state"][:n], non_blocking=True)
            b["box_pin"][:n].copy_(boxes, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        state = b["state_pin"].numpy()[:n]
        rec = b["box_pin"].numpy()[:n].view(_lib.BOX_DTYPE).reshape(-1)
        return dict(bbox=state[:, 1:5].astype(np.int64), score=rec["score"].astype(np.float32), ids=self._ids.copy())

    # ------------------------------------------------------------------ internals
    def _device(self) -> torch.device:
        if not torch.cuda.is_available():
            raise RuntimeError("FEARMultiTracker (H100) needs a CUDA device: there is no CPU path")
        if isinstance(self.cuda_id, int):
            return torch.device("cuda", self.cuda_id)
        dev = torch.device(self.cuda_id)
        if dev.type != "cuda":
            raise RuntimeError(f"FEARMultiTracker (H100) needs a CUDA device, got {self.cuda_id!r}: there is no CPU path")
        return torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())

    def _check_frames(self, frames):
        """-> (list of frames, True if they are CUDA tensors).  Raises ValueError before any device call."""
        if isinstance(frames, (np.ndarray, torch.Tensor)) and frames.ndim == 3:
            frames = [frames]
        frames = list(frames)
        if not frames:
            raise ValueError("no frames given")
        on_device = isinstance(frames[0], torch.Tensor)
        if any(isinstance(f, torch.Tensor) != on_device for f in frames):
            raise ValueError("frames of one call must be all numpy arrays or all CUDA tensors, not a mix")
        for i, f in enumerate(frames):
            if on_device:
                self._check_tensor_frame(i, f)
            elif not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 \
                    or f.shape[0] < 1 or f.shape[1] < 1:
                what = f"{f.dtype} {f.shape}" if isinstance(f, np.ndarray) else type(f).__name__
                raise ValueError(f"frame {i} must be a uint8 HxWx3 RGB array, got {what}")
        return frames, on_device

    def _check_tensor_frame(self, i: int, f: torch.Tensor) -> None:
        if f.dtype != torch.uint8 or f.ndim != 3 or f.shape[2] != 3 or not (1 <= f.shape[0] <= _MAX_SIDE) \
                or not (1 <= f.shape[1] <= _MAX_SIDE):
            raise ValueError(f"frame {i} must be a uint8 HxWx3 RGB tensor, got {f.dtype} {tuple(f.shape)}")
        if min(f.stride()) < 0:
            raise ValueError(f"frame {i} has a negative stride {f.stride()}")
        if f.device.type != "cuda":
            raise ValueError(f"frame {i} is a {f.device} tensor: tensor frames must be on the tracker's CUDA device "
                             "(pass host frames as numpy arrays)")
        dev = self._device()
        if f.device != dev:
            raise ValueError(f"frame {i} is on {f.device}, the tracker on {dev}")

    @staticmethod
    def _check_streams(streams, n: int, num_frames: int) -> np.ndarray:
        s = np.asarray(streams)
        if s.shape != (n,) or (s.size and not np.issubdtype(s.dtype, np.integer)):
            raise ValueError(f"streams must be ({n},) integer frame indices, got {s.dtype} {s.shape}")
        s = s.astype(np.int64)
        if s.size and (s.min() < 0 or s.max() >= num_frames):
            raise ValueError(f"stream indices must be in [0, {num_frames}), got {s.tolist()}")
        return s

    def _buffers(self, dev: torch.device) -> dict:
        b = self._buf
        if b is not None and b["device"] == dev:
            return b
        if b is not None:  # moving to another device: the targets' state and templates do not follow
            raise RuntimeError(f"FEARMultiTracker state lives on {b['device']}, not {dev}")
        m, size = self.max_targets, int(self.tracking_config["instance_size"])
        tsize = int(self.tracking_config["template_size"])
        self._buf = b = dict(
            device=dev,
            state=torch.zeros((m, _lib.TARGET_INTS), dtype=torch.int32, device=dev),
            zf=torch.zeros((m, 256, 8, 8), dtype=torch.float32, device=dev),
            crops=torch.empty((m, size, size, 3), dtype=torch.uint8, device=dev),
            tcrops=torch.empty((m, tsize, tsize, 3), dtype=torch.uint8, device=dev),
            state_pin=torch.empty((m, _lib.TARGET_INTS), dtype=torch.int32).pin_memory(),
            box_pin=torch.empty((m, _lib.BOX_DTYPE.itemsize), dtype=torch.uint8).pin_memory(),
            frames_pin=None, frames=None, views_pin=None, views=None, sums_pin=None, sums=None)
        return b

    def _upload_frames(self, frames, on_device: bool, dev: torch.device) -> None:
        """Write the FearFrameView table of ``frames`` into the device table the kernels read.  Numpy frames are packed
        into the pinned staging buffer first and sent with one host-to-device copy (the packed layout is recomputed
        only when their shapes change); CUDA tensors are used where they are."""
        b, num_frames, rec = self._buf, len(frames), _lib.VIEW_DTYPE.itemsize
        if b["views"] is None or b["views"].numel() < num_frames * rec:  # grows only: the step graph keys on it
            b["views_pin"] = torch.empty(num_frames * rec, dtype=torch.uint8).pin_memory()
            b["views"] = torch.empty(num_frames * rec, dtype=torch.uint8, device=dev)
            # fear_frame_sums_u8 writes uint64; int64 storage, read back as uint64
            b["sums_pin"] = torch.empty((num_frames, 3), dtype=torch.int64).pin_memory()
            b["sums"] = torch.empty((num_frames, 3), dtype=torch.int64, device=dev)
        table = b["views_pin"].numpy()[:num_frames * rec].view(_lib.VIEW_DTYPE)
        if on_device:
            for i, f in enumerate(frames):
                table[i] = frame_view(f)
        else:
            key = tuple(f.shape for f in frames)
            if key != self._frames_key:
                offsets, off = [], 0
                for f in frames:
                    offsets.append(off)
                    off += -(-f.size // _FRAME_ALIGN) * _FRAME_ALIGN
                if b["frames"] is None or b["frames"].numel() < off:
                    b["frames_pin"] = torch.empty(off, dtype=torch.uint8).pin_memory()
                    b["frames"] = torch.empty(off, dtype=torch.uint8, device=dev)
                b["offsets"], b["nbytes"] = offsets, off
                self._frames_key = key
            pin, base = b["frames_pin"].numpy(), b["frames"].data_ptr()
            for i, (f, o) in enumerate(zip(frames, b["offsets"])):
                np.copyto(pin[o:o + f.size].reshape(f.shape), f)
                h, w = f.shape[:2]
                table[i] = (base + o, 3 * w, 3, 1, h, w)
            nb = b["nbytes"]
            b["frames"][:nb].copy_(b["frames_pin"][:nb], non_blocking=True)
        b["views"][:num_frames * rec].copy_(b["views_pin"][:num_frames * rec], non_blocking=True)

    def _step(self, n: int, num_frames: int, dev: torch.device) -> torch.Tensor:
        b, cfg, lib = self._buf, self.tracking_config, _lib.load()
        size = int(cfg["instance_size"])
        s = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.fear_crop_targets_view_u8(b["views"].data_ptr(), num_frames, b["state"].data_ptr(), n,
                                                 float(cfg["search_context"]), size, b["crops"].data_ptr(), s),
                   "fear_crop_targets_view_u8")
        boxes = self.net.track_boxes(b["crops"][:n], b["zf"][:n])
        _lib.check(lib.fear_advance_targets_view(boxes.data_ptr(), b["views"].data_ptr(), num_frames,
                                                 b["state"].data_ptr(), n, size, s), "fear_advance_targets_view")
        return boxes

    def _run_step(self, n: int, num_frames: int, dev: torch.device) -> torch.Tensor:
        """One step, as a CUDA graph after one eager warm-up call (the pattern of FEARTracker's gpu_crop path).  The
        kernels read the frame table when they run, so frame addresses and shapes are not baked into the graph: it is
        keyed by the target count, the frame count, the table buffer and the net's generation.  ``cuda_graph=False``
        in the tracking config keeps eager launches."""
        key = (n, num_frames, self._buf["views"].data_ptr())
        if key != self._graph_key or (self._graph is not None and self._graph_gen != self.net.generation()):
            # new target or frame count, a new table buffer, or the net's workspace / weights / options changed: the
            # pointers and sizes baked into the captured graph are stale -> warm up eagerly and capture again
            self._graph, self._graph_key, self._calls = None, key, 0
        use_graph = self.tracking_config.get("cuda_graph", True) and self._graph_ok
        if use_graph and self._graph is None and self._calls >= 1:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._graph_boxes = self._step(n, num_frames, dev)
                self._graph, self._graph_gen = g, self.net.generation()
            except RuntimeError as exc:
                warnings.warn(f"FEARMultiTracker: CUDA-graph capture of the step failed ({exc}); using eager launches")
                self._graph_ok = False
                torch.cuda.synchronize(dev)
        self._calls += 1
        if use_graph and self._graph is not None:
            self._graph.replay()
            return self._graph_boxes
        return self._step(n, num_frames, dev)
