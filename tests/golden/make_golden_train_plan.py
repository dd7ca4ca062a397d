"""tests/golden/make_golden_train_plan.py -- the training step's launch log of every case of tests/test_train_plan.py.

Replays begin_step, run_forward and the segmented backward of the training engine on the CPU against the test's stand-ins
for the library and CUDA streams, and writes tests/golden/train_plan.json.gz (gzip with mtime 0, so the file depends on the
log only).

    python tests/golden/make_golden_train_plan.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import test_train_plan as tp  # noqa: E402


def main():
    out = {}
    for case in tp.CASES:
        out[case] = tp.replay(case)
        print(case, "calls", len(out[case]["log"]), "launch counts", out[case]["launch_counts"])
    tp.dump(out, tp.FIXTURE)


if __name__ == "__main__":
    main()
