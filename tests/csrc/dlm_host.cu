// Test infrastructure: cv_b200/csrc/device_libm.cuh's sinf_glibc / cosf_glibc compiled as HOST code, so that a machine without a GPU
// can hold the device source to the host libm.  Reads little-endian float32 from stdin, writes sin then cos of each (float32) to
// stdout.  Build: nvcc -std=c++17 -Xcompiler -ffp-contract=off dlm_host.cu
#include <stdio.h>
#include <vector>
#include "../../cv_b200/csrc/device_libm.cuh"

int main() {
    std::vector<float> in;
    float v;
    while (fread(&v, sizeof v, 1, stdin) == 1) in.push_back(v);
    for (float x : in) {
        const float r[2] = {dlm::sinf_glibc(x), dlm::cosf_glibc(x)};
        fwrite(r, sizeof(float), 2, stdout);
    }
    return 0;
}
