"""Generates the squeeze-excite fixtures tests/golden/ser50_objectnav.pt and serx50_imagenav.pt from the UNMODIFIED
reference classes, with make_golden.py's config #3 / #4 recipe (same sensors, rollout, minibatch and recorded outputs)
and an SE backbone.  Run in the build container only:

    python tests/golden/make_golden_se.py [ser50_objectnav] [serx50_imagenav]
"""
from __future__ import annotations

import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as M  # noqa: E402

SE_CASES = {
    # config #3's sensors (rgb, depth, int32 semantic, objectgoal, compass, gps) with SE-ResNet50 and GRU-512
    "ser50_objectnav": dict(T=4, N=2, H=128, W=128, backbone="se_resnet50", rnn="GRU", layers=1, n_actions=6,
                            n_categories=21, imagegoal=False, seed=51),
    # config #4's dual encoder (observation + goal image) with SE-ResNeXt50 and LSTM-512 x 2
    "serx50_imagenav": dict(T=4, N=2, H=128, W=128, backbone="se_resneXt50", rnn="LSTM", layers=2, n_actions=4,
                            n_categories=0, imagegoal=True, seed=61),
}


def main():
    only = sys.argv[1:]
    unknown = [n for n in only if n not in SE_CASES]
    if unknown:
        raise SystemExit(f"unknown case(s) {unknown}; known: {sorted(SE_CASES)}")
    torch.set_num_threads(8)
    M.NEXT_CASES = {n: c for n, c in SE_CASES.items() if not only or n in only}
    M._next_cases(M.ref_shim.ref(), [])


if __name__ == "__main__":
    main()
