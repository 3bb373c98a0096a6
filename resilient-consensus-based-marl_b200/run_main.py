#!/usr/bin/env python
"""Launch the UNMODIFIED reference driver (main.py of mfigura/Resilient-consensus-based-MARL) on the drop-in packages.

    RCMARL_N_ENVS=4096 python resilient-consensus-based-marl_b200/run_main.py /path/to/reference/main.py --H=1 --slow_lr=0.002

`python /path/to/reference/main.py` would put the reference's own directory first on sys.path and import its TensorFlow
agents; this launcher puts the drop-in root first and executes main.py with runpy (which does not add the script's
directory), so `environments`, `agents`, `training`, `tensorflow`, `gym` resolve to this repository."""
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main(argv):
    if len(argv) < 2:
        raise SystemExit(__doc__)
    script = argv[1]
    sys.path.insert(0, HERE)
    sys.argv = [script] + argv[2:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main(sys.argv)
