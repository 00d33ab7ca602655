// cv_b200/csrc/match_wgmma.cuh -- Hamming k-NN on the Hopper tensor cores (wgmma.mma_async u8 x u8 -> s32, accumulators in registers).
// Included by match.cu (uses its mbarrier / bulk-copy helpers and the (distance << 22 | index) key logic).
//
//     hamming(a, b) = |a| + |b| - 2 <a, b>      with descriptors expanded to 512 x u8 in {0, 1}: exact in s32
//
// One CTA = 128 queries x one split of the database, walked in tiles of 128 descriptors; two warpgroups of 64 queries each.
//   A (queries)   : expanded once into registers in the wgmma A-fragment layout (16 k-steps x 4 registers per thread); the
//                   expanded operands never exist in global or shared memory
//   B (database)  : thread 0 stages the PACKED tile (128 x 64 B = 8 KB) with cp.async.bulk into a two-slot ring (mbarrier
//                   completion); all 256 threads expand it into the K-major, non-swizzled operand layout (8 x 16 B core
//                   matrices: offset = (r/8)*4096 + (k/16)*128 + (r%8)*16 + k%16), double buffered, and count its bits
//   MMA           : per tile and warpgroup 16 x wgmma m64n128k32; the expansion of the next tile runs while they execute
//   epilogue      : every thread holds 2 query rows x 32 database columns of the s32 accumulator: distance, running best-K;
//                   the four lanes that share a row merge their lists at the end
// The output format (per-split key lists merged by k_knn_merge) is the one of the other two kernels, so results are identical by
// construction; tests/test_gpu_match.py compares all three bit for bit.
#pragma once

namespace wg {

constexpr int QT = 128, DT = 128, KB = 512;             // queries per CTA, database descriptors per tile, expanded bytes per row
constexpr int THREADS = 256;
constexpr uint32_t OP_BYTES = DT * KB;                   // 64 KB per expanded operand tile
constexpr uint32_t STG_BYTES = DT * 64;                  // 8 KB packed
constexpr uint32_t OFF_B = 0, OFF_STG = 2 * OP_BYTES, OFF_PB = OFF_STG + 2 * STG_BYTES, OFF_BAR = OFF_PB + 2 * 2 * DT * 2;
constexpr uint32_t SMEM = OFF_BAR + 2 * 8;               // 148,496 B: one CTA per SM

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// K-major, no swizzle: leading (K) byte offset 128, stride (8-row group) byte offset 4096
__device__ __forceinline__ uint64_t op_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)(128u >> 4) << 16) | ((uint64_t)(4096u >> 4) << 32);
}
// nibble n -> bytes (bit0, bit1, bit2, bit3): n * 0x00204081 puts bit i at bit 8 i
__device__ __forceinline__ uint32_t nib_bytes(uint32_t n) { return ((n & 0xfu) * 0x00204081u) & 0x01010101u; }

// D (+)= A[regs] * B[smem]^T, u8 x u8 -> s32, M = 64 (one warpgroup), N = 128, K = 32
__device__ __forceinline__ void wgmma_u8_n128(int (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p;\n"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// 256 packed bits (half h of a 64-byte row in shared memory) -> their 256 bytes in {0,1} at the row's place in an operand tile;
// returns their population count
__device__ __forceinline__ uint32_t expand_half_row(const uint8_t *packed_row, uint8_t *op_tile, uint32_t r, uint32_t h) {
    uint8_t *dst = op_tile + (r >> 3) * 4096u + (r & 7u) * 16u;
    const uint4 *src = (const uint4 *)(packed_row + 32u * h);
    uint32_t pc = 0;
#pragma unroll
    for (int q = 0; q < 2; q++) {
        const uint4 w4 = src[q];
        const uint32_t ws[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t w = ws[j];
            pc += __popc(w);
#pragma unroll
            for (int s = 0; s < 2; s++) {           // 16 bits -> one 16-byte K chunk
                const uint32_t b = w >> (16 * s);
                const uint4 o = make_uint4(nib_bytes(b), nib_bytes(b >> 4), nib_bytes(b >> 8), nib_bytes(b >> 12));
                const uint32_t chunk = 16u * h + (uint32_t)(q * 8 + j * 2 + s);      // K chunk 0..31 (bits 16*chunk ..)
                *(uint4 *)(dst + chunk * 128u) = o;
            }
        }
    }
    return pc;
}

// grid = (ceil(n_max / 128), splits); partial[(q * splits + s) * K + i] = key with split-local index
template <int K>
__global__ void __launch_bounds__(THREADS, 1) k_hamming_wgmma(const uint8_t *__restrict__ queries, const uint32_t *__restrict__ n_dev,
                                                              uint32_t n_host, const uint8_t *__restrict__ db,
                                                              const uint32_t *__restrict__ m_dev, uint32_t m_host, uint32_t chunk,
                                                              uint32_t *__restrict__ partial) {
    extern __shared__ __align__(1024) uint8_t sm[];
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host, m = m_dev ? min(*m_dev, m_host) : m_host;
    if (blockIdx.x * QT >= n) return;
    const uint32_t lo = min(blockIdx.y * chunk, m), hi = min(lo + chunk, m), cnt = hi - lo;
    const uint32_t ntiles = (cnt + DT - 1) / DT;
    uint8_t *opB = sm + OFF_B, *stg = sm + OFF_STG;
    uint16_t *s_pb = (uint16_t *)(sm + OFF_PB);              // [slot][half][row]
    uint64_t *bar = (uint64_t *)(sm + OFF_BAR);              // staging slot s full
    const uint32_t tid = threadIdx.x, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const uint32_t q0 = blockIdx.x * QT + (tid >> 7) * 64u + ((tid >> 5) & 3u) * 16u + g;     // rows q0 and q0 + 8
    if (tid == 0) {
        mbar_init(&bar[0], 1); mbar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](uint32_t t) {
        const uint32_t first = t * DT, rows = min((uint32_t)DT, cnt - first);
        mbar_expect_tx(&bar[t & 1], rows * 64u);
        tma_load_1d(stg + (t & 1) * STG_BYTES, db + (size_t)(lo + first) * 64, rows * 64u, &bar[t & 1]);
    };
    if (tid == 0) {
        if (ntiles > 0) issue(0);
        if (ntiles > 1) issue(1);
    }
    // A fragments: k-step j, register 0/1 = rows q0/q0+8 at k = 32j + 4 t4 .. +3, register 2/3 the same at k + 16
    uint32_t a[16][4];
    uint32_t pa0 = 0, pa1 = 0;
    {
        const uint4 *r0 = (const uint4 *)(queries + (size_t)min(q0, n - 1) * 64), *r1 = (const uint4 *)(queries + (size_t)min(q0 + 8, n - 1) * 64);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint4 v0 = r0[i], v1 = r1[i];
            const uint32_t w0[4] = {v0.x, v0.y, v0.z, v0.w}, w1[4] = {v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                pa0 += __popc(w0[j]); pa1 += __popc(w1[j]);
                a[4 * i + j][0] = nib_bytes(w0[j] >> (4 * t4));
                a[4 * i + j][1] = nib_bytes(w1[j] >> (4 * t4));
                a[4 * i + j][2] = nib_bytes(w0[j] >> (16 + 4 * t4));
                a[4 * i + j][3] = nib_bytes(w1[j] >> (16 + 4 * t4));
            }
        }
    }
    // thread tid expands half (tid >> 7) of row (tid & 127) of every tile
    auto expand = [&](uint32_t t) {
        const uint32_t s = t & 1, r = tid & 127u, h = tid >> 7, rows = min((uint32_t)DT, cnt - t * DT);
        mbar_wait(&bar[s], (t >> 1) & 1);
        const uint32_t pc = expand_half_row(stg + s * STG_BYTES + min(r, rows - 1) * 64u, opB + s * OP_BYTES, r, h);
        s_pb[(s * 2 + h) * DT + r] = (uint16_t)pc;
        fence_proxy_async();                // the generic-proxy writes become visible to the tensor cores' reads
    };
    uint32_t best0[K], best1[K];
#pragma unroll
    for (int i = 0; i < K; i++) { best0[i] = 0xffffffffu; best1[i] = 0xffffffffu; }
    int acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0;
    if (ntiles > 0) expand(0);
    __syncthreads();
    if (tid == 0 && ntiles > 2) issue(2);
    for (uint32_t t = 0; t < ntiles; t++) {
        const uint32_t s = t & 1, first = t * DT;
        const uint32_t b_addr = smem_u32(opB + s * OP_BYTES);
        wgmma_fence();
#pragma unroll
        for (uint32_t j = 0; j < KB / 32; j++) wgmma_u8_n128(acc, a[j], op_desc(b_addr + j * 256u), j > 0 ? 1u : 0u);
        wgmma_commit();
        if (t + 1 < ntiles) expand(t + 1);  // the other operand buffer: its last reader (tile t - 1) completed before the barrier below
        wgmma_wait0();
        const uint16_t *pb = s_pb + s * 2 * DT;
#pragma unroll
        for (int i = 0; i < 16; i++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const uint32_t c = 8u * i + 2u * t4 + e, col = first + c;
                if (col < cnt) {
                    const uint32_t p = pb[c] + pb[DT + c];
                    insert_key<K>(best0, ((pa0 + p - 2u * (uint32_t)acc[4 * i + e]) << IDX_BITS) | col);
                    insert_key<K>(best1, ((pa1 + p - 2u * (uint32_t)acc[4 * i + 2 + e]) << IDX_BITS) | col);
                }
            }
        }
        __syncthreads();                    // operand tile t + 1 and its counts are complete; tile t and staging slot t + 1 are free
        if (tid == 0 && t + 3 < ntiles) issue(t + 3);
    }
    // merge the four lanes that share a row
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        uint32_t o0[K], o1[K];
#pragma unroll
        for (int i = 0; i < K; i++) { o0[i] = __shfl_xor_sync(0xffffffffu, best0[i], o); o1[i] = __shfl_xor_sync(0xffffffffu, best1[i], o); }
#pragma unroll
        for (int i = 0; i < K; i++) { insert_key<K>(best0, o0[i]); insert_key<K>(best1, o1[i]); }
    }
    if (t4 == 0) {
        if (q0 < n) {
            uint32_t *out = partial + ((size_t)q0 * gridDim.y + blockIdx.y) * K;
#pragma unroll
            for (int i = 0; i < K; i++) out[i] = best0[i];
        }
        if (q0 + 8 < n) {
            uint32_t *out = partial + ((size_t)(q0 + 8) * gridDim.y + blockIdx.y) * K;
#pragma unroll
            for (int i = 0; i < K; i++) out[i] = best1[i];
        }
    }
}

}  // namespace wg
