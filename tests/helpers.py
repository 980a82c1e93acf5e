"""Shared test helpers (fixture loading + the error metrics SURVEY.md section 7.4 prescribes)."""
import json
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-3  # BASELINE.json north_star: maps within 1e-3 fp32 relative tolerance
# Workspace / guard poison words (tests/poison_check.py): A is a quiet NaN with a payload no kernel emits; B is finite
# (+16 777 218.0) and survives a ReLU, which would turn a NaN read by mistake into 0
POISON_A, POISON_B = 0x7FA5A5A5, 0x4B800001


def load_hotpath_state():
    with np.load(os.path.join(GOLDEN, "fear_xs_hotpath_state.npz")) as f:
        return {k: torch.from_numpy(f[k]) for k in f.files}


def load_full_state():
    """All 520 checkpoint keys: hot-path values from the fixture, the never-executed tail
    (xif5_*, xif6_0, head, num_batches_tracked) zero-filled with the recorded shapes/dtypes."""
    with open(os.path.join(GOLDEN, "state_dict_keys.json")) as f:
        keys = json.load(f)
    hot = load_hotpath_state()
    sd = {}
    for k, (shape, dtype) in keys.items():
        sd[k] = hot[k] if k in hot else torch.zeros(shape, dtype=getattr(torch, dtype))
    return sd


def poison_workspace(net, word=POISON_B):
    """Fill every word of the library workspace of ``net``'s handle with ``word`` (fear_debug_fill_workspace), on the
    current stream: a later call that reads a workspace value it did not write in the same call no longer matches."""
    from feartracker_b200 import _lib

    h, lib = net._ensure_handle(next(net.parameters()).device)
    _lib.check(lib.fear_debug_fill_workspace(h, word, torch.cuda.current_stream().cuda_stream),
               "fear_debug_fill_workspace")


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


def map_errors(a, b):
    """(i) max |a-b| / max(|b|, 1e-3*||b||inf)  and  (ii) ||a-b||inf / ||b||inf, per map."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    binf = np.abs(b).max()
    e1 = (np.abs(a - b) / np.maximum(np.abs(b), 1e-3 * binf)).max()
    e2 = np.abs(a - b).max() / binf
    return float(e1), float(e2)


def assert_maps_close(a, b, what, tol=TOL, inf_tol=None):
    """Both metrics <= tol.  For intermediates pass inf_tol (a tighter bound on the inf-norm error)
    and leave the element-wise bound at the contract tolerance."""
    e1, e2 = map_errors(a, b)
    assert e1 <= tol and e2 <= (tol if inf_tol is None else inf_tol), \
        f"{what}: rel err {e1:.3e} / inf-norm err {e2:.3e} exceeds {tol} / {inf_tol}"
    return e1, e2
