"""Measures cv-sfm's reconstruction export on the device (include/cvb200_export.h) on the scenes of scripts/prof_optimize_reconstruction.py
(32, 128 and 512 views): host-clock medians of cvb_export_reconstruction_dev and cvb_normalize_reconstruction_dev on device-resident
inputs, each call ending in a synchronise; of cvb_export_reconstruction on host arrays (uploads and copies back included); of the host
PLY writer (cv_b200.formats.export_ply) on the exported arrays; and of the C oracle on 8 host threads, which triangulates every landmark
again for each view observing it, as the reference does.  The card's name and power limit are read in the same run.

    python scripts/prof_export_reconstruction.py [--out FILE]    # every row is printed as a JSON line; --out also writes them as one file
"""
import argparse
import ctypes as C
import importlib.util
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("prof_optimize_reconstruction", os.path.join(ROOT, "scripts", "prof_optimize_reconstruction.py"))
P = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(P)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="*", default=[32, 128, 512])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = P.card()
    import torch
    import cv_b200
    from cv_b200._lib import load_export_library
    from cv_b200.export import CAMERA_DTYPE, NORMALIZE_RESULT_DTYPE, ExportSettings, export_reconstruction
    from cv_b200.formats import export_ply
    from oracle import pyoracle_export as X
    ctx = cv_b200.Context(0)
    dev = torch.device("cuda", 0)
    lib, st, tri = load_export_library(), ExportSettings(), cv_b200.LinearEigenTriangulator()
    rows = []
    for V in a.views:
        built = P.build(V)
        s, cons = built[0], built[1]
        snap = (s["poses"], s["view_offsets"], s["view_landmarks"], s["bearings"], s["landmark_offsets"], s["observations"])
        col = np.random.default_rng(0).integers(0, 256, (len(s["view_landmarks"]), 3), dtype=np.uint8)
        t = (lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dt).reshape(-1).copy()).to(dev))
        Pd, vo, vl, bear = t(s["poses"], np.float64), t(s["view_offsets"], np.uint32), t(s["view_landmarks"], np.uint32), t(s["bearings"], np.float64)
        lo, ob, cold = t(s["landmark_offsets"], np.uint32), t(s["observations"], np.uint32), t(col, np.uint8)
        consd = t(np.ascontiguousarray(cons).view(np.uint8), np.uint8)
        Lm, nf, no, Cn = len(s["landmark_offsets"]) - 1, len(s["view_landmarks"]), len(s["observations"]), len(cons)
        pts = torch.zeros(Lm * 3, dtype=torch.float64, device=dev)
        pcol = torch.zeros(Lm * 3, dtype=torch.uint8, device=dev)
        npt = torch.zeros(1, dtype=torch.int32, device=dev)
        cams = torch.zeros(V * CAMERA_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        pout = torch.zeros(V * 12, dtype=torch.float64, device=dev)
        cout = torch.zeros(max(consd.numel(), 1), dtype=torch.uint8, device=dev)
        res = torch.zeros(NORMALIZE_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()

        def export_dev():
            ctx.check(lib.cvb_export_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), V, Pd.data_ptr(), vo.data_ptr(),
                                                        vl.data_ptr(), bear.data_ptr(), cold.data_ptr(), nf, Lm, lo.data_ptr(), ob.data_ptr(),
                                                        no, pts.data_ptr(), pcol.data_ptr(), npt.data_ptr(), cams.data_ptr(), None))

        def normalize_dev():
            ctx.check(lib.cvb_normalize_reconstruction_dev(ctx.handle, C.addressof(st), C.addressof(tri.cfg), V, Pd.data_ptr(), vo.data_ptr(),
                                                           vl.data_ptr(), bear.data_ptr(), nf, Lm, lo.data_ptr(), ob.data_ptr(), no,
                                                           consd.data_ptr(), Cn, 0, pout.data_ptr(), cout.data_ptr(), res.data_ptr()))

        e = export_reconstruction(ctx, *snap, col)
        cams_h = [dict(optical_center=c["optical_center"], up_direction=c["up_direction"], forward_direction=c["forward_direction"],
                       focal_length=c["focal_length"]) for c in e["cameras"]]
        o = X.export_reconstruction(*snap, col, threads=8)
        same = all(np.ascontiguousarray(e[k]).tobytes() == np.ascontiguousarray(o[k]).tobytes() for k in o)
        row = dict(views=V, landmarks=Lm, observations=no, points=len(e["points"]), equal_to_oracle=bool(same),
                   export_dev_ms=1e3 * P.med(export_dev, a.reps), normalize_dev_ms=1e3 * P.med(normalize_dev, a.reps),
                   export_host_form_ms=1e3 * P.med(lambda: export_reconstruction(ctx, *snap, col), a.reps),
                   export_ply_ms=1e3 * P.med(lambda: export_ply(io.StringIO(), list(zip(e["points"], e["colors"])), cams_h, True), 3),
                   oracle_export_8_threads_ms=1e3 * P.med(lambda: X.export_reconstruction(*snap, col, threads=8), 3),
                   oracle_normalize_ms=1e3 * P.med(lambda: X.normalize_reconstruction(*snap, cons), 3))
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(gpu=gpu, rows=rows), f, indent=1)
    print(json.dumps(dict(gpu=gpu)))


if __name__ == "__main__":
    main()
