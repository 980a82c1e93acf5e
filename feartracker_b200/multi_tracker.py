"""FEARMultiTracker: many targets, in one or several video streams, stepped together once per frame.

    trk = FEARMultiTracker(net, cuda_id=0, max_targets=64, **FEAR_XS_TRACKER_KWARGS)
    ids = trk.add(frames, rects, streams=None)   # frames: one HxWx3 uint8 array or a list of F; streams -> frame index
    out = trk.update(frames)                      # {"bbox": (N,4) int64, "score": (N,) float32, "ids": (N,) int64}
    trk.remove(ids); trk.reset()

Every target behaves exactly like its own ``FEARTracker(gpu_crop=True)`` started on the same frame with the same
rect: the rect is clamped, the padding colour is the mean colour of the init frame, the template is the network
features of its 128 x 128 context crop, and each frame runs crop -> network -> decode -> rescale -> clamp.  Instead of
one batch-1 step and one host round trip per target, one step runs all N targets at batch N:

    fear_crop_targets_u8 (N search crops)  ->  fear_track_u8 (B = N, Bz = N)  ->  fear_advance_targets

on per-target state kept in device memory (an (N, 16) int32 tensor of FearTarget records, include/fear_b200.h), so the
step is captured once as a CUDA graph and replayed every frame; the host packs the frames into one pinned buffer, sends
them with one copy and reads back the boxes and scores.  The launch count of a step does not depend on N.
"""
import math
import warnings
from typing import Any, Dict, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib, image_ops

_FRAME_ALIGN = 16  # byte alignment of each frame inside the packed buffer


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
        self._frames_key = None  # frame shapes the packed buffer and the frame table are laid out for
        self._epoch = 0  # bumped whenever the packed frame buffer or the frame table moves
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
        current frame is ``frames[streams[i]]``.  Returns the new targets' ids."""
        frames = self._check_frames(frames)
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
        pads = {}
        for i, (rect, s) in enumerate(zip(rects, streams)):
            frame = frames[s]
            box = image_ops.clamp_bbox(rect, frame.shape)
            ctx = image_ops.context_box(box, cfg["template_bbox_offset"])
            inner = image_ops.trim_box([box[0] - ctx[0], box[1] - ctx[1], box[2], box[3]], (ctx[3], ctx[2]))
            if inner[2] * inner[3] == 0:
                raise IndexError("target box has zero area inside its context crop")
            if s not in pads:  # cv::saturate_cast of the float64 mean colour, as FEARTracker's padding
                pads[s] = np.clip(np.rint(np.mean(frame, axis=(0, 1))), 0, 255).astype(np.int32)
            recs[i, 0] = s
            recs[i, 1:5] = box
            recs[i, 9:12] = pads[s]
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            self._upload_frames(frames, dev)
            lib = _lib.load()
            n0 = len(self._ids)
            stream = torch.cuda.current_stream(dev)
            b["state"][n0:n0 + n].copy_(torch.from_numpy(recs).pin_memory(), non_blocking=True)
            size = int(cfg["template_size"])
            crops = b["tcrops"][:n]
            _lib.check(lib.fear_crop_targets_u8(b["frames"].data_ptr(), b["table"].data_ptr(), len(frames),
                                                b["state"][n0].data_ptr(), n, float(cfg["template_bbox_offset"]),
                                                size, crops.data_ptr(), stream.cuda_stream), "fear_crop_targets_u8")
            b["zf"][n0:n0 + n].copy_(self.net.get_features(crops))
            stream.synchronize()  # the pinned staging buffer is reused by the next call
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
        """One frame of every stream -> the new box and score of every target, in the order of ``ids``."""
        frames = self._check_frames(frames)
        n = len(self._ids)
        if n and int(self._streams.max()) >= len(frames):
            raise ValueError(f"targets track stream {int(self._streams.max())} but only {len(frames)} frames were given")
        if n == 0:
            return dict(bbox=np.zeros((0, 4), dtype=np.int64), score=np.zeros(0, dtype=np.float32),
                        ids=self._ids.copy())
        dev = self._device()
        with torch.cuda.device(dev):
            b = self._buffers(dev)
            self._upload_frames(frames, dev)
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

    @staticmethod
    def _check_frames(frames):
        if isinstance(frames, np.ndarray) and frames.ndim == 3:
            frames = [frames]
        frames = list(frames)
        if not frames:
            raise ValueError("no frames given")
        for i, f in enumerate(frames):
            if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 \
                    or f.shape[0] < 1 or f.shape[1] < 1:
                what = f"{f.dtype} {f.shape}" if isinstance(f, np.ndarray) else type(f).__name__
                raise ValueError(f"frame {i} must be a uint8 HxWx3 RGB array, got {what}")
        return frames

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
            frames_pin=None, frames=None, table=None)
        return b

    def _upload_frames(self, frames, dev: torch.device) -> None:
        """Pack the frames into the pinned staging buffer and send them with one host-to-device copy.  The buffer and
        the frame table are laid out again only when the frame shapes change."""
        b = self._buf
        key = tuple(f.shape for f in frames)
        if key != self._frames_key:
            table = np.zeros(len(frames), dtype=_lib.FRAME_DTYPE)
            off = 0
            for i, f in enumerate(frames):
                table[i] = (off, f.shape[0], f.shape[1])
                off += -(-f.size // _FRAME_ALIGN) * _FRAME_ALIGN
            if b["frames"] is None or b["frames"].numel() < off:
                b["frames_pin"] = torch.empty(off, dtype=torch.uint8).pin_memory()
                b["frames"] = torch.empty(off, dtype=torch.uint8, device=dev)
            b["table"] = torch.from_numpy(table.view(np.uint8).copy()).to(dev)
            b["offsets"] = [int(o) for o in table["offset"]]
            b["nbytes"] = off
            self._frames_key = key
            self._epoch += 1
        pin = b["frames_pin"].numpy()
        for f, o in zip(frames, b["offsets"]):
            np.copyto(pin[o:o + f.size].reshape(f.shape), f)
        nb = b["nbytes"]
        b["frames"][:nb].copy_(b["frames_pin"][:nb], non_blocking=True)

    def _step(self, n: int, num_frames: int, dev: torch.device) -> torch.Tensor:
        b, cfg, lib = self._buf, self.tracking_config, _lib.load()
        size = int(cfg["instance_size"])
        s = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.fear_crop_targets_u8(b["frames"].data_ptr(), b["table"].data_ptr(), num_frames,
                                            b["state"].data_ptr(), n, float(cfg["search_context"]), size,
                                            b["crops"].data_ptr(), s), "fear_crop_targets_u8")
        boxes = self.net.track_boxes(b["crops"][:n], b["zf"][:n])
        _lib.check(lib.fear_advance_targets(boxes.data_ptr(), b["table"].data_ptr(), num_frames, b["state"].data_ptr(),
                                            n, size, s), "fear_advance_targets")
        return boxes

    def _run_step(self, n: int, num_frames: int, dev: torch.device) -> torch.Tensor:
        """One step, as a CUDA graph after one eager warm-up call (the pattern of FEARTracker's gpu_crop path).  The
        graph is keyed by the target count, the frame layout and the net's generation; ``cuda_graph=False`` in the
        tracking config keeps eager launches."""
        key = (n, self._frames_key, self._epoch)
        if key != self._graph_key or (self._graph is not None and self._graph_gen != self.net.generation()):
            # new target set or frame layout, or the net's workspace / weights / options changed: the pointers and
            # sizes baked into the captured graph are stale -> warm up eagerly and capture again
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
