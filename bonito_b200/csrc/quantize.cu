// fp16 -> int8 quantisation of activations for the INT8 input projection (--quantize; the reference's counterpart is koi's
// int8 LSTM path, bonito/crf/model.py:245, bonito/cli/basecaller.py:186-189).  LSTM inputs are outputs of tanh / o*tanh(c),
// i.e. inside (-1, 1): a fixed scale of 127 needs no calibration.  HBM-bound: 2 B in, 1 B out per element.
#include "common.cuh"

namespace {

__global__ void __launch_bounds__(256)
quantize_i8_kernel(const __half* __restrict__ x, int8_t* __restrict__ out, long long n8, float scale) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(x) + i);
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    int q[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 f = __half22float2(h[k]);
        q[2 * k] = max(-127, min(127, __float2int_rn(f.x * scale)));
        q[2 * k + 1] = max(-127, min(127, __float2int_rn(f.y * scale)));
    }
    uint2 o;
    o.x = (uint32_t)(q[0] & 255) | ((uint32_t)(q[1] & 255) << 8) | ((uint32_t)(q[2] & 255) << 16) | ((uint32_t)(q[3] & 255) << 24);
    o.y = (uint32_t)(q[4] & 255) | ((uint32_t)(q[5] & 255) << 8) | ((uint32_t)(q[6] & 255) << 16) | ((uint32_t)(q[7] & 255) << 24);
    reinterpret_cast<uint2*>(out)[i] = o;
}

// chunk(): overlapping windows of one read, gathered (and converted to fp16) on the device -- the arithmetic of
// bonito.util.chunk (bonito/util.py:142-161): a read shorter than a chunk is tiled up to the chunk size; otherwise windows of
// `chunksize` every `chunksize - overlap` samples starting at stub = (length - overlap) % step, preceded by one window over
// signal[:chunksize] when stub > 0.
template <typename T>
__global__ void __launch_bounds__(256)
chunk_kernel(const T* __restrict__ signal, long long length, int chunksize, int step, int stub, __half* __restrict__ out,
             long long row_stride) {
    const int c = blockIdx.y;
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= chunksize) return;
    long long src;
    if (length < chunksize) src = j % length;
    else if (stub > 0) src = (c == 0 ? 0 : (long long)stub + (long long)(c - 1) * step) + j;
    else src = (long long)c * step + j;
    out[(long long)c * row_stride + j] = __float2half_rn((float)signal[src]);
}

}  // namespace

// number of chunks bonito.util.chunk returns for a read of `length` samples (chunksize > 0)
int chunk_count(long long length, int chunksize, int overlap) {
    if (length < chunksize) return 1;
    const int step = chunksize - overlap;
    const long long stub = (length - overlap) % step;
    return (int)((length - stub - chunksize) / step + 1 + (stub > 0 ? 1 : 0));
}

int launch_chunk_signal(const void* signal, int is_f32, long long length, int chunksize, int overlap, __half* out,
                        long long row_stride, cudaStream_t stream) {
    B200_REQUIRE(length > 0 && chunksize > 0 && overlap >= 0 && overlap < chunksize && row_stride >= chunksize,
                 "chunk_signal: bad geometry (length %lld, chunksize %d, overlap %d)", length, chunksize, overlap);
    const int n = chunk_count(length, chunksize, overlap), step = chunksize - overlap;
    B200_REQUIRE(n <= 65535, "chunk_signal: at most 65535 chunks per read (%d): the chunk index is gridDim.y", n);
    const int stub = length < chunksize ? 0 : (int)((length - overlap) % step);
    const dim3 grid((unsigned)((chunksize + 255) / 256), (unsigned)n);
    if (is_f32) chunk_kernel<float><<<grid, 256, 0, stream>>>((const float*)signal, length, chunksize, step, stub, out, row_stride);
    else chunk_kernel<__half><<<grid, 256, 0, stream>>>((const __half*)signal, length, chunksize, step, stub, out, row_stride);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_quantize_i8(const __half* x, int8_t* out, long long n, float scale, cudaStream_t stream) {
    B200_REQUIRE(n % 8 == 0 && ((uintptr_t)x % 16) == 0 && ((uintptr_t)out % 8) == 0,
                 "quantize_i8: the element count must be a multiple of 8 and the buffers 16 / 8-byte aligned");
    const long long n8 = n / 8;
    if (n8 == 0) return 0;
    quantize_i8_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(x, out, n8, scale);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
