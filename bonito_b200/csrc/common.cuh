// Shared device/host helpers for the bonito_b200 sm_90a kernels.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// ---------------------------------------------------------------------------
// error plumbing: every C-ABI entry point returns 0 / negative and records a
// message retrievable through b200_last_error().
// ---------------------------------------------------------------------------
void b200_set_error(const char* fmt, ...);

#define B200_CHECK_CUDA(expr)                                                            \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            b200_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                           __FILE__, __LINE__);                                          \
            return -1;                                                                   \
        }                                                                                \
    } while (0)

#define B200_REQUIRE(cond, ...)                                                          \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            b200_set_error(__VA_ARGS__);                                                 \
            return -2;                                                                   \
        }                                                                                \
    } while (0)

// activation codes (B200_ACT_*) are shared with the C ABI
#include "../../include/bonito_b200.h"

// ---------------------------------------------------------------------------
// device math with the reference's fp16 rounding points
// ---------------------------------------------------------------------------
__device__ __forceinline__ float round_f16(float x) { return __half2float(__float2half_rn(x)); }

// sigmoid / tanh from one ex2 and one rcp each (2 SFU ops, no IEEE division): abs error ~2e-7, far below fp16
// resolution (the single-op tanh.approx is ~5e-4, too coarse for 1e-3 parity).
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// the bare SFU instruction: exp2f() wraps it in a rescaling path for results below 2^-126, which every use here adds to 1
// (or multiplies into a sum that is >= 1), so flushing those to zero changes nothing
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoid_f(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float tanh_f(float x) {
    return fmaf(2.0f, rcp_approx(1.0f + ex2_approx(-2.8853900817779268f * x)), -1.0f);
}

__device__ __forceinline__ float swish_f(float x) { return x * sigmoid_f(x); }

// sigma(i), sigma(f), tanh(g), sigma(o) from four ex2 and ONE reciprocal (batch inversion); the exponent arguments are
// clamped so the product of the four denominators stays finite (sigma(-20.8) = 9e-10: the clamp is invisible in fp16).
__device__ __forceinline__ void gate_activations(float ai, float af, float ag, float ao, float& si, float& sf, float& tg,
                                                 float& so) {
    constexpr float L = 1.4426950408889634f, CLAMP = 30.0f;
    const float di = 1.0f + ex2_approx(fminf(-L * ai, CLAMP));
    const float df = 1.0f + ex2_approx(fminf(-L * af, CLAMP));
    const float dg = 1.0f + ex2_approx(fminf(-2.0f * L * ag, CLAMP));
    const float dO = 1.0f + ex2_approx(fminf(-L * ao, CLAMP));
    const float pif = di * df, pgo = dg * dO;
    const float r = rcp_approx(pif * pgo);
    const float rif = r * pgo, rgo = r * pif;
    si = rif * df;
    sf = rif * di;
    tg = fmaf(2.0f, rgo * dO, -1.0f);
    so = rgo * dg;
}

// Apply an epilogue activation to a value that the reference would already have
// rounded to fp16 (conv/linear output), then round again (elementwise op output).
__device__ __forceinline__ float apply_act_f16(float v, int act, float lo, float hi) {
    v = round_f16(v);
    switch (act) {
        case B200_ACT_SWISH: return round_f16(swish_f(v));
        case B200_ACT_TANH: return round_f16(tanh_f(v));
        case B200_ACT_CLAMP: return fminf(fmaxf(v, lo), hi);
        case B200_ACT_SCALE: return round_f16(v * lo);
        case B200_ACT_TANH_SCALE: return round_f16(round_f16(tanh_f(v)) * lo);
        case B200_ACT_SWISH_CLAMP: return fminf(fmaxf(round_f16(swish_f(v)), lo), hi);
        case B200_ACT_RELU: return fmaxf(v, 0.f);
        default: return v;
    }
}

// ---------------------------------------------------------------------------
// small PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src, bool valid) {
    uint32_t d = smem_u32(smem_dst);
    int bytes = valid ? 16 : 0;  // src-size 0 => zero fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gmem_src), "r"(bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}

// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Row remap applied by GEMM epilogues: input row r -> (outer, inner) = divmod(r, rows_inner);
// rows with inner >= valid_inner are dropped; output row = inner*stride_inner + outer*stride_outer, or, with a second
// level (group > 0): (outer2, outer1) = divmod(outer, group), output row = inner*stride_inner + outer1*stride_outer +
// outer2*stride_group  (chunk -> (tile, chunk in tile) or (tile, frame) splits of the tile layout).
struct RowMap {
    int rows_inner;
    int valid_inner;
    long long stride_inner;
    long long stride_outer;
    int group;
    long long stride_group;
};

__device__ __forceinline__ long long map_row(const RowMap& m, int r) {
    int outer = r / m.rows_inner;
    int inner = r - outer * m.rows_inner;
    if (inner >= m.valid_inner) return -1;
    long long o = (long long)inner * m.stride_inner;
    if (m.group > 0) {
        const int outer2 = outer / m.group;
        o += (long long)outer2 * m.stride_group;
        outer -= outer2 * m.group;
    }
    return o + (long long)outer * m.stride_outer;
}

struct GemmEpilogue {
    const __half* bias;  // [N] or nullptr
    int act;             // B200_ACT_*
    float lo, hi;        // clamp bounds
    RowMap map;
    // column blocks: output column c of mapped row R goes to row R + (c / cb_width) * cb_rows, column c % cb_width
    // (cb_width = 0: off).  Used to write the LSTM input projection as [t][cluster rank][chunk][256 columns].
    int cb_width, cb_rows;
};

// Host-side launchers (defined in the .cu files, used by abi.cu)
int chunk_count(long long length, int chunksize, int overlap);
int launch_chunk_signal(const void* signal, int is_f32, long long length, int chunksize, int overlap, __half* out,
                        long long row_stride, cudaStream_t stream);
int launch_gemm_mma(const __half* A, long long lda, const __half* B, __half* C, long long ldc, int M, int N, int K,
                    const GemmEpilogue& ep, cudaStream_t stream);
int launch_gemm_tc(const __half* A, long long lda, const __half* B, __half* C, long long ldc, int M, int N, int K,
                   const GemmEpilogue& ep, int max_ctas, cudaStream_t stream);
