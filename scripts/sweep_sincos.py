"""Exhaustive check of the full-range sin / cos: every one of the 2^32 float32 inputs through
  - dlm::sinf_glibc / cosf_glibc (cv_b200/csrc/device_libm.cuh) compiled as host code with -ffp-contract=off, and
  - the describe oracle's ref_full_sinf / ref_full_cosf (oracle/ref_stages.c),
against the host libm's sinf / cosf (glibc 2.39 on x86-64 is the reference: Rust's f32::sin / cos call it).  Equal bits, or NaN on
both sides, count as a match.  CPU only, under a minute on 8 cores (OpenMP); builds into a temporary directory.
python scripts/sweep_sincos.py"""
import os
import platform
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SRC = r'''
#include <math.h>
#include <stdio.h>
#include <string.h>
#include "cv_b200/csrc/device_libm.cuh"
extern "C" float ref_full_sinf(float);
extern "C" float ref_full_cosf(float);
static inline bool same(float a, float b) {
    uint32_t x, y;
    memcpy(&x, &a, 4); memcpy(&y, &b, 4);
    return x == y || (a != a && b != b);
}
int main() {
    unsigned long long dev_bad = 0, ora_bad = 0;
#pragma omp parallel for reduction(+ : dev_bad, ora_bad) schedule(static, 1 << 16)
    for (long long i = 0; i < (1ll << 32); i++) {
        const uint32_t u = (uint32_t)i;
        float x;
        memcpy(&x, &u, 4);
        const float s = sinf(x), c = cosf(x);
        dev_bad += !(same(dlm::sinf_glibc(x), s) && same(dlm::cosf_glibc(x), c));
        ora_bad += !(same(ref_full_sinf(x), s) && same(ref_full_cosf(x), c));
    }
    printf("device_libm.cuh: %llu mismatching inputs of 2^32\nref_stages.c:    %llu mismatching inputs of 2^32\n", dev_bad, ora_bad);
    return dev_bad || ora_bad;
}
'''


def main():
    with tempfile.TemporaryDirectory() as tmp:
        cu = os.path.join(tmp, "sweep.cu")
        open(cu, "w").write(SRC)
        obj = os.path.join(tmp, "ref_stages.o")
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-c",
                               os.path.join(ROOT, "oracle", "ref_stages.c"), "-o", obj])
        exe = os.path.join(tmp, "sweep")
        subprocess.check_call([NVCC, "-std=c++17", "-O2", "-I" + ROOT, "-Xcompiler", "-fopenmp,-ffp-contract=off", cu, obj, "-o", exe,
                               "-lgomp", "-lm"])
        libc = platform.libc_ver()
        print(f"host libm: {libc[0]} {libc[1]}", flush=True)
        sys.exit(subprocess.call([exe]))


if __name__ == "__main__":
    main()
