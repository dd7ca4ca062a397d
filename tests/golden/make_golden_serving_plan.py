"""tests/golden/make_golden_serving_plan.py -- the serving pipelines' call log of every case of tests/test_serving_plan.py.

Replays the pipelines on the CPU against the test's stand-ins for the library, CUDA streams, events and graphs, with the
host conv planner at H100 SXM properties, and writes tests/golden/serving_plan.json.gz (gzip with mtime 0, so the file
depends on the log only).

    python tests/golden/make_golden_serving_plan.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import test_serving_plan as tp  # noqa: E402


def main():
    out = {}
    for case in tp.CASES:
        out[case] = tp.replay(case)
        print(case, "calls", len(out[case]))
    tp.dump(out, tp.FIXTURE)


if __name__ == "__main__":
    main()
