"""tests/golden/make_golden_loss_plan.py -- the library calls of every case of tests/test_loss_plan.py.

Replays the detection losses' host code (anchor-free, anchor-aided and self-distillation) on the CPU against the test's
stand-ins for the library and writes tests/golden/loss_plan.json.gz (gzip with mtime 0, so the file depends on the log only).

    python tests/golden/make_golden_loss_plan.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import test_loss_plan as lp  # noqa: E402


def main():
    out = {}
    for case in lp.CASES:
        out[case] = lp.replay(case)
        print(case, "calls", len(out[case]), [e["fn"] for e in out[case]])
    lp.dump(out, lp.FIXTURE)


if __name__ == "__main__":
    main()
