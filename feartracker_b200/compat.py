"""Config / CLI glue so the reference's ``demo_video.py`` (reference demo_video.py:1-62) and any script written against
``model_training.*`` run UNMODIFIED on the H100 implementation, on a machine that has none of hydra / omegaconf /
fire / imageio installed (this image) and no reference package on the path.

Two pieces:

* a minimal Hydra-1.1-style composer -- ``load_hydra_config_from_path(config_path, config_name, overrides)`` with the
  signature and result of reference model_training/utils/hydra.py:33-39 (``initialize`` + ``compose`` +
  ``OmegaConf.to_container(resolve=True)``): a primary YAML with a ``defaults`` list of ``- group: option`` entries,
  ``# @package _global_`` headers, ``${a.b}`` interpolation, dotted ``key=value`` / ``group=option`` overrides; and
  ``instantiate(config, *args, **kwargs)`` (``hydra.utils.instantiate``) resolving ``_target_`` recursively;
* ``install()``: registers stand-in modules in ``sys.modules`` -- ``model_training.model.fear_net`` /
  ``.tracker.fear_tracker`` / ``.dataset.box_coder`` / ``.utils.{torch,hydra,constants}`` mapped onto
  feartracker_b200, plus ``hydra.utils``, ``fire`` and ``imageio.v3`` (cv2-backed) -- each ONLY when the real module
  is not importable.  After that ``_target_: model_training.model.fear_net.FEARNet`` in the reference's own YAML tree
  instantiates the H100 FEARNet.

Not a general Hydra: no config groups inside groups, no sweeps, no resolvers besides plain key interpolation (the
``hydra:`` node, whose ``${now:...}`` needs one, is dropped from the result exactly as ``compose()`` drops it).
"""
import importlib
import os
import re
import sys
import types
from typing import Any, Dict, List, Optional

_INTERP = re.compile(r"\$\{([^${}]+)\}")


# ------------------------------------------------------------------------------------------ composer
def _read_yaml(path: str):
    import yaml

    with open(path, "r") as f:
        text = f.read()
    m = re.match(r"\s*#\s*@package\s+(\S+)", text)
    return (yaml.safe_load(text) or {}), (m.group(1) if m else None)


def _merge(dst: Dict[str, Any], src: Dict[str, Any]) -> Dict[str, Any]:
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = v
    return dst


def _set_dotted(cfg: Dict[str, Any], key: str, value: Any) -> None:
    parts = key.split(".")
    for p in parts[:-1]:
        cfg = cfg.setdefault(p, {})
    cfg[parts[-1]] = value


def _get_dotted(cfg: Dict[str, Any], key: str) -> Any:
    cur = cfg
    for p in key.split("."):
        if not isinstance(cur, dict) or p not in cur:
            raise KeyError(f"interpolation key '{key}' not found")
        cur = cur[p]
    return cur


def _resolve(node: Any, root: Dict[str, Any], depth: int = 0) -> Any:
    if depth > 16:
        raise ValueError("interpolation cycle")
    if isinstance(node, dict):
        return {k: _resolve(v, root, depth) for k, v in node.items()}
    if isinstance(node, list):
        return [_resolve(v, root, depth) for v in node]
    if isinstance(node, str):
        whole = _INTERP.fullmatch(node)
        if whole:  # "${model.stride}" keeps the referenced value's type
            return _resolve(_get_dotted(root, whole.group(1).strip()), root, depth + 1)
        if _INTERP.search(node):
            return _INTERP.sub(lambda m: str(_resolve(_get_dotted(root, m.group(1).strip()), root, depth + 1)), node)
    return node


def compose(config_dir: str, config_name: str, overrides: Optional[List[str]] = None) -> Dict[str, Any]:
    import yaml

    overrides = list(overrides or [])
    primary, _ = _read_yaml(os.path.join(config_dir, config_name + ".yaml"))
    defaults = primary.pop("defaults", []) or []
    choice = {}
    order = []
    for item in defaults:
        if item == "_self_":
            order.append("_self_")
        elif isinstance(item, dict):
            (group, option), = item.items()
            group = group.replace("override ", "").strip()
            choice[group] = option
            order.append(group)
        elif isinstance(item, str):
            order.append(("file", item))
    value_overrides = []
    for ov in overrides:
        key, _, val = ov.partition("=")
        key = key.lstrip("+")
        if key in choice or os.path.isdir(os.path.join(config_dir, key)):
            if key not in choice:
                order.append(key)
            choice[key] = val
        else:
            value_overrides.append((key, yaml.safe_load(val)))
    if "_self_" not in order:
        order.insert(0, "_self_")  # Hydra 1.1: without _self_ the primary config is composed first
    cfg: Dict[str, Any] = {}
    for entry in order:
        if entry == "_self_":
            _merge(cfg, primary)
            continue
        if isinstance(entry, tuple):
            node, pkg = _read_yaml(os.path.join(config_dir, entry[1] + ".yaml"))
            _merge(cfg, node)
            continue
        option = choice[entry]
        if option is None or (entry.startswith("hydra/")):
            continue  # "group: null" selects nothing; hydra/* plugin groups are not part of the job config
        node, pkg = _read_yaml(os.path.join(config_dir, entry, str(option) + ".yaml"))
        if pkg == "_global_":
            _merge(cfg, node)
        else:
            target = cfg
            for p in (pkg or entry).split("/" if pkg is None else "."):
                target = target.setdefault(p, {})
            _merge(target, node)
    for key, val in value_overrides:
        _set_dotted(cfg, key, val)
    cfg.pop("hydra", None)  # compose() returns the job config without the hydra node
    return _resolve(cfg, cfg)


def load_hydra_config_from_path(config_path: str, config_name: str, overrides=None) -> Dict[str, Any]:
    """Same call as reference model_training/utils/hydra.py:33-39; ``config_path`` is relative to the working
    directory (or absolute), the result is a plain resolved dict."""
    if isinstance(overrides, dict):
        overrides = [f"{k}={v}" for k, v in overrides.items()]
    return compose(os.path.abspath(config_path), config_name, overrides)


def _locate(path: str):
    module, _, attr = path.rpartition(".")
    if not module:
        raise ImportError(f"_target_ '{path}' is not a dotted path")
    return getattr(importlib.import_module(module), attr)


def instantiate(config: Any, *args, **kwargs):
    """``hydra.utils.instantiate``: call ``_target_`` with the remaining keys (+ overrides); nested nodes carrying
    their own ``_target_`` are instantiated first (Hydra 1.1 ``_recursive_`` default)."""
    if config is None:
        return None
    if not isinstance(config, dict) or "_target_" not in config:
        raise ValueError("instantiate needs a config with a _target_ key")
    params = {k: v for k, v in config.items() if k not in ("_target_", "_recursive_", "_convert_", "_partial_")}
    params.update(kwargs)
    for k, v in list(params.items()):
        if isinstance(v, dict) and "_target_" in v:
            params[k] = instantiate(v)
    return _locate(config["_target_"])(*args, **params)


# ------------------------------------------------------------------------------------------ module shims
def _importable(name: str) -> bool:
    if name in sys.modules:
        return True
    try:
        importlib.import_module(name)
        return True
    except Exception:
        return False


def _module(name: str, **attrs) -> types.ModuleType:
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__feartracker_b200_shim__ = True
    sys.modules[name] = m
    return m


def _fire(fn):
    """fire.Fire(main): ``--name=value`` / ``--name value`` flags parsed with yaml (lists, ints, ...)."""
    import yaml

    argv, kwargs, i = sys.argv[1:], {}, 0
    while i < len(argv):
        a = argv[i]
        if not a.startswith("--"):
            raise SystemExit(f"unexpected argument {a!r}")
        key, eq, val = a[2:].partition("=")
        if not eq:
            i += 1
            val = argv[i] if i < len(argv) else "true"
        kwargs[key.replace("-", "_")] = yaml.safe_load(val)
        i += 1
    return fn(**kwargs)


def _make_imageio_v3():
    import cv2
    import numpy as np

    def imread(path, **_):
        cap = cv2.VideoCapture(str(path))
        frames = []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            frames.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
        cap.release()
        if not frames:
            raise IOError(f"cannot decode {path}")
        return np.stack(frames)

    def immeta(path, **_):
        cap = cv2.VideoCapture(str(path))
        fps = cap.get(cv2.CAP_PROP_FPS) or 25.0
        cap.release()
        return {"fps": fps}

    def imwrite(path, frames, fps=25.0, **_):
        frames = list(frames)
        h, w = frames[0].shape[:2]
        out = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), float(fps), (w, h))
        for f in frames:
            out.write(cv2.cvtColor(np.ascontiguousarray(f), cv2.COLOR_RGB2BGR))
        out.release()

    return dict(imread=imread, immeta=immeta, imwrite=imwrite)


def install(force: bool = False) -> List[str]:
    """Register the stand-in modules (see the module docstring); returns the names that were registered."""
    import feartracker_b200 as fb
    from . import box_coder, constants, fear_net, tracker

    done = []

    def shim(name, **attrs):
        if force or not _importable(name):
            _module(name, **attrs)
            done.append(name)

    if force or not _importable("model_training"):
        for pkg in ("model_training", "model_training.model", "model_training.tracker", "model_training.utils",
                    "model_training.dataset"):
            _module(pkg, __path__=[])
            done.append(pkg)
        _module("model_training.model.fear_net", FEARNet=fear_net.FEARNet)
        _module("model_training.model.blocks", Encoder=fear_net.Encoder, AdjustLayer=fear_net.AdjustLayer,
                BoxTower=fear_net.BoxTower)
        _module("model_training.tracker.fear_tracker", FEARTracker=tracker.FEARTracker)
        _module("model_training.tracker.base_tracker", Tracker=tracker.Tracker, TrackingState=tracker.TrackingState)
        sys.modules["model_training.tracker"].Tracker = tracker.Tracker
        _module("model_training.dataset.box_coder", FEARBoxCoder=box_coder.FEARBoxCoder,
                TrackerDecodeResult=box_coder.TrackerDecodeResult)
        _module("model_training.utils.constants", TARGET_CLASSIFICATION_KEY=constants.TARGET_CLASSIFICATION_KEY,
                TARGET_REGRESSION_LABEL_KEY=constants.TARGET_REGRESSION_LABEL_KEY)
        _module("model_training.utils.torch", load_from_lighting=fb.load_from_lighting)
        _module("model_training.utils.hydra", load_hydra_config_from_path=load_hydra_config_from_path)
        done += ["model_training.model.fear_net", "model_training.tracker.fear_tracker", "model_training.utils.torch",
                 "model_training.utils.hydra"]
    if force or not _importable("hydra"):
        _module("hydra", __path__=[])
        _module("hydra.utils", instantiate=instantiate)
        done.append("hydra.utils")
    shim("fire", Fire=_fire)
    if force or not _importable("imageio"):
        _module("imageio", __path__=[])
        _module("imageio.v3", **_make_imageio_v3())
        done.append("imageio.v3")
    return done
