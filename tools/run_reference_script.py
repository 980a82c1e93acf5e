#!/usr/bin/env python
"""Run a script written against the reference package (e.g. the reference's demo_video.py) UNMODIFIED on the H100
implementation: installs feartracker_b200.compat's stand-ins for ``model_training.*`` / hydra / fire / imageio (each
only if the real module is missing), then executes the script as ``__main__``.

    cd <dir containing model_training/config and the video/checkpoint paths the script expects>
    python tools/run_reference_script.py <reference>/demo_video.py --output_path=/tmp/out.mp4
"""
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    from feartracker_b200 import compat

    names = compat.install()
    print(f"[feartracker_b200.compat] stand-ins registered: {', '.join(names) or 'none'}", file=sys.stderr)
    script = sys.argv[1]
    sys.argv = [script] + sys.argv[2:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
