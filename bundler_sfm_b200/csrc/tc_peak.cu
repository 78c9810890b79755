// tc_peak.cu -- measured int8 tensor-pipe ceiling of this GPU: a plain wgmma.mma_async u8 x u8 -> s32 loop.  One CTA per
// SM, two warpgroups, each issuing back-to-back M64 N128 K32 MMAs (K = 4 x 32 per tile; n_tile = 256 issues two N = 128
// halves into two register accumulators, like the MATCH search kernel) on operand tiles resident in shared memory -- a ring
// of four (A, B) tile pairs of pseudo-random bytes, K-major SWIZZLE_128B like the real kernel, so consecutive tiles read
// different operands; no loads, no epilogue.  What it reports is the rate the MATCH search kernel is measured against
// (bench.py roofline.peak); it is an upper bound for any kernel built from the same instruction shape.
#include "common.h"
#include "tc_ptx.cuh"
#include <atomic>

namespace bsfm {
using namespace bsfm::ptx;

template <int N_TILE>
__global__ void __launch_bounds__(256, 1) i8_peak_kernel(int iters, unsigned *sink)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    const uint32_t base = (raw_addr + 1023u) & ~1023u;
    uint8_t *smem = smem_raw + (base - raw_addr);
    constexpr int STAGES = 4, STAGE_BYTES = 16384 + 32768;      // ring of (A 128 x 128 B, B 256 x 128 B) tiles, as a pipelined GEMM keeps
    for (int q = threadIdx.x; q < STAGES * STAGE_BYTES / 4; q += blockDim.x) {      // pseudo-random operand bytes
        uint32_t v = (uint32_t) q * 2654435761u + blockIdx.x * 40503u;
        v ^= v >> 15; v *= 2246822519u; v ^= v >> 13;
        reinterpret_cast<uint32_t *>(smem)[q] = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy writes of the tiles -> async proxy (MMA) reads
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    uint32_t d0[64], d1[64];
#pragma unroll
    for (int i = 0; i < 64; i++) { d0[i] = 0; d1[i] = 0; }
    for (int it = 0; it < iters; it++) {
        const uint32_t st = base + (uint32_t) (it & (STAGES - 1)) * STAGE_BYTES;      // every tile reads different operands
        const uint64_t ad = make_sw128_desc(st + wg * 8192), bd = make_sw128_desc(st + 16384);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; kk++) wgmma_u8_n128(d0, ad + (uint64_t) (kk * 2), bd + (uint64_t) (kk * 2), 1u);
        if (N_TILE == 256) {
#pragma unroll
            for (int kk = 0; kk < 4; kk++) wgmma_u8_n128(d1, ad + (uint64_t) (kk * 2), bd + (uint64_t) (1024 + kk * 2), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();      // bound the number of MMA groups in flight
    }
    wgmma_wait<0>();
    wgmma_fence_regs(d0);
    wgmma_fence_regs(d1);
    unsigned x = 0;
#pragma unroll
    for (int i = 0; i < 64; i++) x ^= d0[i] ^ d1[i];
    if (x == 0x9e3779b9u) sink[0] = x;      // keeps the accumulators (and so the MMAs) alive
}

}  // namespace bsfm

// Runs the loop and returns the measured rate in TOP/s (2 ops per multiply-add), < 0 on error.  n_tile = 128 or 256.
extern "C" double bsfm_measure_int8_peak(int n_tile, int iters)
{
    using namespace bsfm;
    clear_error();
    if (require_device() != BSFM_OK) return -1.0;
    if ((n_tile != 128 && n_tile != 256) || iters < 16) { set_error("bsfm_measure_int8_peak: n_tile must be 128 or 256, iters >= 16"); return -1.0; }
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) { set_error("device query failed"); return -1.0; }
    const size_t smem = 4 * (16384 + 32768) + 1024;
    void (*kern)(int, unsigned *) = (n_tile == 256) ? i8_peak_kernel<256> : i8_peak_kernel<128>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) != cudaSuccess) { set_error("cudaFuncSetAttribute failed"); return -1.0; }
    unsigned *sink = nullptr;
    if (cudaMalloc(&sink, sizeof(unsigned)) != cudaSuccess) { set_error("cudaMalloc failed"); return -1.0; }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    kern<<<sms, 256, smem>>>(iters / 8 + 16, sink);      // warm-up
    cudaEventRecord(e0);
    kern<<<sms, 256, smem>>>(iters, sink);
    cudaEventRecord(e1);
    count_launch(2);
    float ms = 0.f;
    const cudaError_t e = cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(sink);
    if (e != cudaSuccess || ms <= 0.f) { set_error("bsfm_measure_int8_peak: %s", cudaGetErrorString(e)); return -1.0; }
    const double ops = (double) sms * iters * 4.0 * (128.0 * n_tile * 32.0) * 2.0;
    return ops / (ms * 1e-3) / 1e12;
}

// ---- fp64 issue rates (dev measurement behind DESIGN.md's notes on the Cholesky pivot chain) ----
// mode 0: vector DFMA, 8 independent chains per thread;  mode 1: DMMA m8n8k4, 4 independent accumulator pairs per thread;
// mode 2: DMMA m16n8k8 (the Cholesky trailing update's shape), 4 independent accumulator quads per thread.
// One CTA per SM, `warps` warps; returns SM cycles per warp instruction per SM sub-partition (warps spread over the 4 of them).
namespace bsfm {
__global__ void fp64_rate_kernel(int iters, int mode, double *sink, unsigned long long *cycles)
{
    double a[16];
#pragma unroll
    for (int i = 0; i < 16; i++) a[i] = 1.0 + 1e-9 * (threadIdx.x + i);
    const double b = 1.0 + 1e-12 * threadIdx.x, c = 1e-13;
    __syncthreads();
    const unsigned long long t0 = clock64();
    if (mode == 0) {
        for (int it = 0; it < iters; it++) {
#pragma unroll
            for (int i = 0; i < 8; i++) a[i] = fma(a[i], b, c);
        }
    } else if (mode == 1) {
        for (int it = 0; it < iters; it++) {
#pragma unroll
            for (int i = 0; i < 8; i += 2)
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(a[i]), "+d"(a[i + 1]) : "d"(b), "d"(c));
        }
    } else {
        for (int it = 0; it < iters; it++) {
#pragma unroll
            for (int i = 0; i < 16; i += 4)
                asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %4, %5}, {%4, %5}, {%0, %1, %2, %3};"
                             : "+d"(a[i]), "+d"(a[i + 1]), "+d"(a[i + 2]), "+d"(a[i + 3]) : "d"(b), "d"(c));
        }
    }
    const unsigned long long t1 = clock64();
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += a[i];
    if (s == 12345.678) sink[0] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) cycles[0] = t1 - t0;
}
}  // namespace bsfm

extern "C" double bsfm_measure_fp64_issue_cycles(int mode, int warps, int iters)
{
    using namespace bsfm;
    clear_error();
    if (require_device() != BSFM_OK) return -1.0;
    if (warps < 1 || warps > 32 || iters < 16 || (mode < 0 || mode > 2)) { set_error("bsfm_measure_fp64_issue_cycles: bad arguments"); return -1.0; }
    double *sink = nullptr; unsigned long long *cyc = nullptr, h = 0;
    if (cudaMalloc(&sink, 8) != cudaSuccess || cudaMalloc(&cyc, 8) != cudaSuccess) { set_error("cudaMalloc failed"); return -1.0; }
    fp64_rate_kernel<<<1, 32 * warps>>>(iters, mode, sink, cyc);
    fp64_rate_kernel<<<1, 32 * warps>>>(iters, mode, sink, cyc);
    count_launch(2);
    const cudaError_t e = cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    cudaFree(sink); cudaFree(cyc);
    if (e != cudaSuccess) { set_error("bsfm_measure_fp64_issue_cycles: %s", cudaGetErrorString(e)); return -1.0; }
    const double instr_per_warp = (double) iters * (mode == 0 ? 8.0 : 4.0);
    const double warps_per_smsp = (warps + 3) / 4;
    return (double) h / (instr_per_warp * warps_per_smsp);
}
