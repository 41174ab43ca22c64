#!/usr/bin/env python
"""Generates tests/golden/detect_plane_fit.npz from the UNMODIFIED reference (oracle/_ref/libref_mtrack.so, built by
oracle/build_ref.py from the reference sources): detect + reEstimateThresh with DetectorPlaneFitSize 1, 3 and 4 on the
small_frames() pair, the threshold chained as in tests/flow.py.  Each window size runs in a process of its own
(tests/plane_fit.py).  The other golden files are not touched.

    python tests/golden/make_plane_fit_golden.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from flow import DOG_THRESH, POS_NEG, SMALL, small_frames  # noqa: E402
from oracle import build_ref  # noqa: E402
from plane_fit import ref_detect_child  # noqa: E402

RADII = (1, 3, 4)

if __name__ == "__main__":
    assert build_ref.build(level_b=False), "reference sources not available"
    f0, f1 = small_frames()
    out = {}
    with tempfile.TemporaryDirectory() as td:
        for R in RADII:
            c = SMALL
            r = ref_detect_child(td, np.stack([f0, f1]), R, c["cam"], c["sigma0"], c["ksigma"], c["thresh"], c["kl_max"],
                                 c["kl_ref"], c["gain"], c["tmax"], c["tmin"], POS_NEG, DOG_THRESH, c["track_points"])
            for i in range(2):
                out["r%d_f%d_kn_tresh" % (R, i)] = r["f%d_kn_tresh" % i]
                out["r%d_f%d_kl" % (R, i)] = r["f%d_kl" % i].view(np.uint8)
                out["r%d_f%d_mask" % (R, i)] = r["f%d_mask" % i]
            print("R=%d kn/tresh:" % R, r["f0_kn_tresh"], r["f1_kn_tresh"])
    np.savez_compressed(os.path.join(HERE, "detect_plane_fit.npz"), **out)
    print("wrote detect_plane_fit.npz")
