// desc_offset.cu -- how does wgmma apply the swizzle to an A descriptor whose 8-row groups start off the
// swizzle pattern's boundary (the column kernel's tap operands, conv_col.cu)?
//
//   nvcc -std=c++17 -O2 -gencode arch=compute_90a,code=sm_90a -I pvnet_b200/csrc \
//        -o benchmarks/micro/desc_offset benchmarks/micro/desc_offset.cu && benchmarks/micro/desc_offset
//
// A tile of 160 rows is written in TMA's swizzled layout (32-, 64- or 128-byte rows) at a 1024-byte aligned
// address; one m64n32k8 MMA reads 64 rows of it through a descriptor that starts at row 0..15 with 8-row
// groups `pitch` rows apart, against one-hot weights, so the output is the operand itself.  Each line counts
// the starts (and K steps) whose output differs from the expected rows, for three base-offset settings:
// 0, the start address's bits 7-9, and the start row's phase.  `dirty` sets the 13 low mantissa bits of
// every operand: the expected values are the truncated ones.  Every descriptor stays inside the tile.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "ptx.cuh"

__device__ __forceinline__ float aval(int R, int k, int dirty)
{
    uint32_t h = (uint32_t)R * 2654435761u ^ (uint32_t)k * 40503u;
    h ^= h >> 13;
    float v = (float)(1024 + (h & 1023));
    uint32_t b = __float_as_uint(v);
    if (dirty) b |= 0x1FFFu;
    return __uint_as_float(b);
}

__global__ void probe(int rowb, int pitch, int start_row, int ks, int base_mode, int dirty, int *bad)
{
    extern __shared__ uint8_t raw[];
    uint8_t *sm = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
    const int NR = 160;
    uint8_t *sA = sm, *sB = sm + NR * 128;
    const int kc = rowb / 4;
    for (int i = threadIdx.x; i < NR * kc; i += blockDim.x) {
        int R = i / kc, k = i % kc;
        *reinterpret_cast<float *>(sA + ptx::swizzle_off((uint32_t)(R * rowb + k * 4), rowb)) = aval(R, k, dirty);
    }
    for (int i = threadIdx.x; i < 32 * kc; i += blockDim.x) {
        int n = i / kc, k = i % kc;
        *reinterpret_cast<float *>(sB + ptx::swizzle_off((uint32_t)(n * rowb + k * 4), rowb)) = (n < 8 && n == k % 8) ? 1.f : 0.f;
    }
    ptx::fence_proxy_async();
    __syncthreads();
    const uint32_t a_start = ptx::smem_u32(sA) + (uint32_t)(start_row * rowb);
    uint64_t base = 0;
    if (base_mode == 1) base = (a_start >> 7) & 7;
    if (base_mode == 2) base = start_row & 7;
    const uint64_t layout = rowb == 128 ? 1ull : (rowb == 64 ? 2ull : 3ull);
    const uint64_t ad = (uint64_t)(((a_start + 32u * ks) & 0x3ffff) >> 4) | (1ull << 16) |
                        ((uint64_t)((pitch * rowb) >> 4) << 32) | (base << 49) | (layout << 62);
    const uint64_t bd = ptx::make_kmajor_desc(ptx::smem_u32(sB), rowb) + (uint64_t)(2 * ks);
    float d[16];
    for (int i = 0; i < 16; ++i) d[i] = -1.f;
    ptx::wgmma_fence();
    ptx::Wgmma<32>::ss(d, ad, bd, 0u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(d);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    int nb = 0;
    for (int j = 0; j < 4; ++j)
        for (int e = 0; e < 4; ++e) {
            const int m = 16 * warp + g + 8 * (e >> 1), n = 8 * j + 2 * t + (e & 1);
            float exp = 0.f;
            if (n < 8) {
                const int R = start_row + (m / 8) * pitch + (m % 8);
                exp = __uint_as_float(__float_as_uint(aval(R, 8 * ks + n, dirty)) & 0xFFFFE000u);
            }
            if (d[4 * j + e] != exp) ++nb;
        }
    atomicAdd(bad, nb);
}

int main()
{
    int *bad;
    cudaMalloc(&bad, sizeof(int));
    cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    const int rowbs[3] = {32, 64, 128}, pitches[3] = {10, 11, 16};
    for (int dirty = 0; dirty < 2; ++dirty)
        for (int ri = 0; ri < 3; ++ri)
            for (int pi = 0; pi < 3; ++pi)
                for (int bm = 0; bm < 3; ++bm) {
                    const int rowb = rowbs[ri], pitch = pitches[pi];
                    int tot = 0, fails = 0, cases = 0;
                    char first[256] = "";
                    for (int sr = 0; sr < 16; ++sr)
                        for (int ks = 0; ks < rowb / 32; ++ks) {
                            cudaMemset(bad, 0, sizeof(int));
                            probe<<<1, 128, 64 * 1024>>>(rowb, pitch, sr, ks, bm, dirty, bad);
                            int h = 0;
                            cudaError_t e = cudaMemcpy(&h, bad, sizeof(int), cudaMemcpyDeviceToHost);
                            if (e != cudaSuccess) {
                                printf("cuda error %s\n", cudaGetErrorString(e));
                                return 1;
                            }
                            ++cases;
                            tot += h;
                            if (h) {
                                if (!fails) snprintf(first, sizeof first, "first fail start_row %d ks %d (%d bad)", sr, ks, h);
                                ++fails;
                            }
                        }
                    printf("dirty %d rowb %3d pitch %2d base_mode %d: %3d/%3d cases fail, %6d bad entries %s\n", dirty, rowb,
                           pitch, bm, fails, cases, tot, first);
                }
    cudaFree(bad);
    return 0;
}
