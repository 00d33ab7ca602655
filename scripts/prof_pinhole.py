"""Kernel time of cv-pinhole on the device (include/cvb200_pinhole.h) from the per-kernel CUDA events of cvb_ctx_profile, over warmed
launches: the pose reprojection error of 200 000 matches with each of the six triangulators (one shared pose), EssentialMatrix residuals
of 64 matrices x 5 000 matches, and recondition / decompose of 4 096 matrices.  Reads the card's name and power limit in the same run.
Prints one line per configuration and one JSON line.
python scripts/prof_pinhole.py [launches]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv_b200  # noqa: E402
from cv_b200 import pinhole as P  # noqa: E402
from tests.geom_util import two_view_scene  # noqa: E402
from tests.pinhole_cases import essential_batch  # noqa: E402

LAUNCHES = max(10, int(sys.argv[1]) if len(sys.argv) > 1 else 20)
TRIS = [cv_b200.LinearEigenTriangulator, cv_b200.SineL1Triangulator, cv_b200.MeanMeanTriangulator, cv_b200.RelativeDltTriangulator,
        cv_b200.AngularL1Triangulator, cv_b200.AngularLInfinityTriangulator]

ctx = cv_b200.Context(0)
rows = []


def run(name, kernel, call, **shape):
    call()                                              # warm-up: module load, workspace allocation
    ctx.sync()
    ctx.profile(True)
    for _ in range(LAUNCHES):
        call()
    ctx.sync()
    rep = ctx.profile_report()
    ctx.profile(False)
    ms = rep[kernel]["ms"] / rep[kernel]["launches"]
    rows.append(dict(name=name, kernel=kernel, kernel_ms=ms, launches=rep[kernel]["launches"], **shape))
    print(f"{name:28s} {kernel:26s} {ms:9.4f} ms/launch  {shape}")


R, t, a, b, _ = two_view_scene(np.random.default_rng(200), 200_000, outlier_frac=0.2, noise=1e-4)
for cls in TRIS:
    tri = cls()
    run(f"reprojection {cls.__name__}", "k_pose_reprojection_error", lambda: P._reprojection([(R, t)], a, b, tri, ctx), n=len(a))
Es = essential_batch(np.random.default_rng(64), 4096)
run("residuals_essential", "k_residuals_essential", lambda: P.residuals_essential(Es[:64], a[:5000], b[:5000], ctx), m=64, n=5000)
run("recondition", "k_essential_recondition", lambda: P.essential_recondition_batch(Es, 1e-12, 1000, ctx), m=len(Es))
run("decompose", "k_essential_decompose", lambda: P.essential_decompose_batch(Es, 1e-12, 1000, ctx), m=len(Es))
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"card: {gpu}")
print(json.dumps(dict(card=gpu, launches=LAUNCHES, rows=rows)))
