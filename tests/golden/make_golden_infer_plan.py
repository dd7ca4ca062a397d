"""tests/golden/make_golden_infer_plan.py -- the inference forward's launch log of every case of tests/test_infer_plan.py.

Replays the engine's forwards on the CPU against the test's stand-ins for the library and CUDA streams, with the host conv
planner at H100 SXM properties, and writes tests/golden/infer_plan.json.gz (gzip with mtime 0, so the file depends on the log
only).

    python tests/golden/make_golden_infer_plan.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import test_infer_plan as tp  # noqa: E402


def main():
    out = {}
    for case in tp.CASES:
        out[case] = tp.replay(case)
        print(case, "calls", len(out[case]["log"]), "streams", out[case]["streams"], "events", out[case]["events"],
              "launch count", out[case].get("launch_count"))
    tp.dump(out, tp.FIXTURE)


if __name__ == "__main__":
    main()
