"""The fused detector response (`k_detector_response`: Lx, Ly, Ldet and the extrema mask in one pass per octave) and the
three separate kernels it replaces (`CVB_NO_FUSE_DET=1`) both match the oracle stage by stage and give the same keypoints."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(no_fuse):
    code = ("import hashlib; from tests.common import kitti_frame; from tests.test_gpu_akaze import _compare_all; "
            "k, d = _compare_all(kitti_frame('0000000000'), 0.001); "
            "print(len(d), hashlib.sha1(d.tobytes() + k.tobytes()).hexdigest())")
    env = dict(os.environ)
    env.pop("CVB_NO_FUSE_DET", None)
    if no_fuse:
        env["CVB_NO_FUSE_DET"] = "1"
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stdout.strip()


def test_fused_and_unfused_detector_response_agree():
    fused, unfused = _run(False), _run(True)
    assert fused.startswith("3425 ") and fused == unfused, (fused, unfused)
