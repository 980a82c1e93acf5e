"""FEARBoxCoder: score/regression maps -> boxes, executed by libfear_b200's decode kernel.

Mirror of reference model_training/dataset/box_coder.py:14-107 (``decode``; ``encode`` builds
training labels and is outside the inference hot path).
"""
from collections import namedtuple
from typing import Any, Dict, Union

import numpy as np
import torch

from . import _lib
from .fear_net import _make_grid

TrackerDecodeResult = namedtuple("TrackerDecodeResult", ["bbox", "pred_coords"])


def search_geometry_supported(score_size, total_stride, instance_size) -> bool:
    """Whether libfear_b200 runs this tracking geometry: a square search of side S, a multiple of 16 in [16, 256],
    stride 16 and S / 16 score cells per side (FEAR-XS is (16, 16, 256))."""
    try:
        s, t, size = int(score_size), int(total_stride), int(instance_size)
    except (TypeError, ValueError):
        return False
    if (s, t, size) != (score_size, total_stride, instance_size):
        return False
    return t == 16 and size % 16 == 0 and 16 <= size <= 256 and s == size // 16


class FEARBoxCoder:
    def __init__(self, tracker_config: Dict[str, Any]) -> None:
        self.tracker_config = tracker_config
        geometry = (tracker_config["score_size"], tracker_config["total_stride"], tracker_config["instance_size"])
        if not search_geometry_supported(*geometry):
            raise NotImplementedError("libfear_b200 decodes (score_size, total_stride, instance_size) = (S / 16, 16, S) "
                                      f"for S a multiple of 16 in [16, 256]; got {geometry}")
        self.score_size, self.instance_size = int(geometry[0]), int(geometry[2])
        self.grid_x, self.grid_y = _make_grid(self.score_size, 16, self.instance_size)

    def to_device(self, device: Union[str, int]) -> "FEARBoxCoder":
        if device != "cpu" and torch.cuda.is_available():
            self.grid_x, self.grid_y = self.grid_x.to(device), self.grid_y.to(device)
        return self

    def encode(self, bboxes):
        raise NotImplementedError("label encoding belongs to the training pipeline (out of the hot-path scope)")

    @torch.no_grad()
    def decode_records(self, regression_map: torch.Tensor, classification_map: torch.Tensor,
                       use_sigmoid: bool = True) -> np.ndarray:
        """Structured array (x, y, w, h float64; score; row; col; flat) per frame."""
        if not (regression_map.is_cuda and classification_map.is_cuda):
            raise RuntimeError("FEARBoxCoder.decode (H100) needs CUDA tensors: there is no CPU path")
        reg = regression_map.detach().float().contiguous()
        cls = classification_map.detach().float().contiguous()
        b, s = reg.shape[0], self.score_size
        if tuple(reg.shape) != (b, 4, s, s) or cls.numel() != b * s * s:
            raise ValueError(f"decode expects (B,4,{s},{s}) / (B,1,{s},{s}), got {tuple(reg.shape)} / {tuple(cls.shape)}")
        lib = _lib.init(reg.device.index if reg.device.index is not None else torch.cuda.current_device())
        boxes = torch.empty((b, _lib.BOX_DTYPE.itemsize), device=reg.device, dtype=torch.uint8)
        _lib.check(lib.fear_decode_sized(reg.data_ptr(), cls.data_ptr(), b, s, int(use_sigmoid), boxes.data_ptr(),
                                         torch.cuda.current_stream(reg.device).cuda_stream), "fear_decode_sized")
        return boxes.cpu().numpy().view(_lib.BOX_DTYPE).reshape(-1)

    def decode(self, regression_map: torch.Tensor, classification_map: torch.Tensor,
               use_sigmoid: bool = True) -> TrackerDecodeResult:
        rec = self.decode_records(regression_map, classification_map, use_sigmoid)
        bbox = torch.from_numpy(np.stack([rec["x"], rec["y"], rec["w"], rec["h"]], axis=1))  # float64 (B,4)
        return TrackerDecodeResult(bbox=bbox, pred_coords=[(int(r), int(c)) for r, c in zip(rec["row"], rec["col"])])
