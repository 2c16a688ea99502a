// extern "C" surface of libbonito_b200.so (declared in include/bonito_b200.h).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/bonito_b200.h"
#include "common.cuh"

int launch_conv_stem(const __half* x, int N, int L, int C1, int K1, const __half* w1, const __half* b1, int act1,
                     int C2, int K2, const __half* w2, const __half* b2, int act2, __half* out, int Lp, int padl,
                     float lo1, float hi1, float lo2, float hi2, cudaStream_t stream);
int lstm_rec_cluster_size(int H);
int launch_lstm_rec(const __half* gx, const __half* whh, __half* y, int T, int N, int H, int reverse,
                    cudaStream_t stream);
int launch_conv_first(const __half* x, int N, int L, int C, int K, const __half* w, const __half* bias, int act,
                      __half* out, int Lp, int padl, cudaStream_t stream);
int launch_conv_first_ex(const __half* x, int N, int L, int C, int K, int S, const __half* w, const __half* bias, int act,
                         float lo, float hi, __half* out, long long ldo, int Lp, int padl, cudaStream_t stream);
int launch_depthwise(const __half* x, long long ldx, const __half* w, __half* y, long long ldy, int N, int T, int C, int K,
                     cudaStream_t stream);
int launch_ctc_head(const __half* x, long long M, int F, const __half* w, const __half* bias, __half* logp, uint8_t* labels,
                    float* probs, cudaStream_t stream);
size_t sw_align_workspace_bytes(int n_pairs, int max_ref_len);
int launch_sw_align(const uint8_t* query, const long long* query_off, const int* query_len, const uint8_t* ref,
                    const long long* ref_off, const int* ref_len, int n_pairs, void* workspace, int* out, cudaStream_t stream);
size_t pair_align_trace_bytes(int mode, int m, int n, int band);
size_t pair_align_workspace_bytes(int mode, int n_pairs, const int* query_len, const int* ref_len, const int* band,
                                  int traceback);
int launch_pair_align(int mode, const uint8_t* query, const long long* query_off, const int* query_len, const uint8_t* ref,
                      const long long* ref_off, const int* ref_len, const int* band, int n_pairs, int traceback,
                      void* workspace, uint8_t* ops, const long long* ops_off, int* out, cudaStream_t stream);
int launch_rmsnorm_residual(const __half* a, const __half* x, const __half* w, float alpha, float eps, __half* out,
                            long long M, int D, cudaStream_t stream);
int launch_swiglu(const __half* h, __half* out, long long M, int F, cudaStream_t stream);
int launch_attention(__half* qkv, const __half* cos_sin, __half* out, int N, int T, int NH, int head_dim, int wl,
                     int wr, cudaStream_t stream);
int lstm_rec_tile_chunks(int hidden);
int lstm_rec_tile_cluster(int hidden);
int launch_lstm_rec_tile(const __half* gx, const __half* whh, __half* y, void* workspace, int T, int N, int hidden,
                         int reverse, cudaStream_t stream);
size_t lstm_rec_tile_workspace_bytes(int N);
int launch_lstm_fused_tile(const __half* x, const __half* wih, const __half* bias, const __half* whh, __half* y,
                           void* workspace, int T, int N, int hidden, int reverse, cudaStream_t stream);
int lstm_rec_wide_ctas(int hidden);
size_t lstm_rec_wide_workspace_bytes(int N, int hidden);
size_t lstm_rec_wide_status_offset(int N, int hidden);
int lstm_rec_wide_max_chunks(int hidden);
int lstm_rec_wide_resident(int hidden);
int launch_lstm_rec_wide(const __half* gx, const __half* whh, __half* y, void* workspace, int T, int N, int hidden,
                         int reverse, cudaStream_t stream);
size_t crf_decode_workspace_bytes(int N, int T, int state_len);
int launch_crf_decode(const __half* scores, int N, int T, int state_len, float blank, float qscale, float qbias,
                      void* workspace, uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream);
int launch_crf_decode_lb(const __half* scores, int N, int T, int state_len, float qscale, float qbias, void* workspace,
                         uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream);

// one message buffer per host thread: the reference drives this path from background threads (bonito/multiprocessing.py:118-122),
// so a failing call must read back its own message, not another thread's
int launch_crf_beam_search(const __half* scores, int N, int T, int state_len, float blank, int width, float cut, float qscale,
                           float qbias, void* workspace, uint8_t* moves, uint8_t* seq, uint8_t* qual, cudaStream_t stream);

int launch_lstm_crf_fwd(const b200_lstm_crf_plan* p, const __half* x, __half* scores, cudaStream_t stream);
int launch_lstm_stack(const b200_lstm_crf_plan* p, int first, int count, cudaStream_t stream);

size_t ctc_crf_sparse_workspace_bytes(int N, int T, int state_len, int semiring);
size_t ctc_crf_target_workspace_bytes(int N, int T, int L, int semiring);
int ctc_crf_target_max_states();
int launch_ctc_crf_sparse_fwd(const float* scores, int T, int N, int state_len, int semiring, float* logz, float* alpha,
                              void* workspace, cudaStream_t stream);
int launch_ctc_crf_sparse_bwd(const float* scores, int T, int N, int state_len, int semiring, float* beta,
                              cudaStream_t stream);
int launch_ctc_crf_sparse_grad(const float* scores, int T, int N, int state_len, int semiring, const float* g,
                               void* workspace, float* grad, cudaStream_t stream);
int launch_ctc_crf_target_fwd(const float* stay, const float* move, const int* lengths, int T, int N, int L, int semiring,
                              float* logz, void* workspace, cudaStream_t stream);
int launch_ctc_crf_target_grad(const float* stay, const float* move, const int* lengths, int T, int N, int L, int semiring,
                               const float* g, void* workspace, float* dstay, float* dmove, cudaStream_t stream);

size_t ctc_beam_workspace_bytes(int n_reads, long long total_frames, int beam_width);
int launch_ctc_beam_search(const __half* logp, const long long* frame_off, const int* frame_len, int n_reads, int beam_width,
                           float threshold, float qscale, float qbias, void* workspace, size_t workspace_bytes,
                           uint8_t* sequence, uint8_t* qstring, uint8_t* moves, cudaStream_t stream);

int launch_quantize_i8(const __half* x, int8_t* out, long long n, float scale, cudaStream_t stream);
int launch_gemm_i8(const int8_t* A, long long lda, const int8_t* B, const float* col_scale, __half* C, long long ldc, int M,
                   int N, int K, const GemmEpilogue& ep, int max_ctas, cudaStream_t stream);

static thread_local char g_err[1024] = "";

void b200_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" {

int b200_version(void) { return 100; }

const char* b200_last_error(void) { return g_err; }

int b200_conv_stem_fwd(const void* x, int n, int l, int c1, int k1, const void* w1, const void* b1, int act1,
                       int c2, int k2, const void* w2, const void* b2, int act2, void* out, int lp, int padl,
                       void* stream) {
    return b200_conv_stem_fwd_ex(x, n, l, c1, k1, w1, b1, act1, 0.f, 0.f, c2, k2, w2, b2, act2, 0.f, 0.f, out, lp, padl,
                                 stream);
}

int b200_conv_stem_fwd_ex(const void* x, int n, int l, int c1, int k1, const void* w1, const void* b1, int act1, float lo1,
                          float hi1, int c2, int k2, const void* w2, const void* b2, int act2, float lo2, float hi2, void* out,
                          int lp, int padl, void* stream) {
    B200_REQUIRE(x && w1 && w2 && out, "conv_stem: null pointer argument");
    B200_REQUIRE(n >= 0 && l > 0 && lp >= padl + l, "conv_stem: bad sizes n=%d l=%d lp=%d padl=%d", n, l, lp, padl);
    if (n == 0) return 0;
    return launch_conv_stem((const __half*)x, n, l, c1, k1, (const __half*)w1, (const __half*)b1, act1, c2, k2,
                            (const __half*)w2, (const __half*)b2, act2, (__half*)out, lp, padl, lo1, hi1, lo2, hi2,
                            (cudaStream_t)stream);
}

int b200_gemm_fwd(const void* a, long long lda, const void* b, const void* bias, void* c, long long ldc, int m,
                  int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                  long long stride_inner, long long stride_outer, int impl, void* stream) {
    return b200_gemm_fwd_ex(a, lda, b, bias, c, ldc, m, n, k, act, lo, hi, rows_inner, valid_inner, stride_inner,
                            stride_outer, 0, 0, 0, 0, impl, 0, stream);
}

int b200_gemm_fwd_ex(const void* a, long long lda, const void* b, const void* bias, void* c, long long ldc, int m,
                     int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                     long long stride_inner, long long stride_outer, int group, long long stride_group, int cb_width,
                     int cb_rows, int impl, int max_ctas, void* stream) {
    B200_REQUIRE(a && b && c, "gemm: null pointer argument");
    B200_REQUIRE(m >= 0 && n > 0 && k > 0 && rows_inner > 0 && group >= 0, "gemm: bad sizes m=%d n=%d k=%d", m, n, k);
    B200_REQUIRE(k % 8 == 0 && lda % 8 == 0 && n % 8 == 0 && ldc % 8 == 0,
                 "gemm: k, lda, n, ldc must be multiples of 8 (k=%d lda=%lld n=%d ldc=%lld)", k, lda, n, ldc);
    B200_REQUIRE(cb_width >= 0 && cb_rows >= 0 && cb_width % 32 == 0 && (cb_width == 0 || act != B200_ACT_SWIGLU),
                 "gemm: column blocks must be multiples of 32 columns and cannot be combined with SwiGLU (cb_width=%d)",
                 cb_width);
    if (act == B200_ACT_SWIGLU)
        B200_REQUIRE(n % 64 == 0 && !bias && impl != B200_GEMM_MMA_SYNC,
                     "gemm: the fused SwiGLU epilogue needs n %% 64 == 0, no bias and the wgmma path (n=%d)", n);
    B200_REQUIRE(impl == B200_GEMM_AUTO || impl == B200_GEMM_TCGEN05 || impl == B200_GEMM_MMA_SYNC, "gemm: unknown impl %d", impl);
    if (m == 0) return 0;
    GemmEpilogue ep;
    ep.bias = (const __half*)bias;
    ep.act = act;
    ep.lo = lo;
    ep.hi = hi;
    ep.map.rows_inner = rows_inner;
    ep.map.valid_inner = valid_inner;
    ep.map.stride_inner = stride_inner;
    ep.map.stride_outer = stride_outer;
    ep.map.group = group;
    ep.map.stride_group = stride_group;
    ep.cb_width = cb_width;
    ep.cb_rows = cb_rows;
    if (impl == B200_GEMM_AUTO) {
        const char* env = getenv("B200_GEMM_IMPL");
        impl = (env && strcmp(env, "mma") == 0 && act != B200_ACT_SWIGLU) ? B200_GEMM_MMA_SYNC : B200_GEMM_TCGEN05;
    }
    if (impl == B200_GEMM_MMA_SYNC)
        return launch_gemm_mma((const __half*)a, lda, (const __half*)b, (__half*)c, ldc, m, n, k, ep,
                               (cudaStream_t)stream);
    return launch_gemm_tc((const __half*)a, lda, (const __half*)b, (__half*)c, ldc, m, n, k, ep, max_ctas,
                          (cudaStream_t)stream);
}

int b200_conv_first_fwd(const void* x, int n, int l, int c, int k, const void* w, const void* bias, int act, void* out,
                        int lp, int padl, void* stream) {
    B200_REQUIRE(x && w && out, "conv_first: null pointer argument");
    B200_REQUIRE(n >= 0 && l > 0 && lp >= padl + l, "conv_first: bad sizes n=%d l=%d lp=%d padl=%d", n, l, lp, padl);
    if (n == 0) return 0;
    return launch_conv_first((const __half*)x, n, l, c, k, (const __half*)w, (const __half*)bias, act, (__half*)out, lp,
                             padl, (cudaStream_t)stream);
}

int b200_conv_first_fwd_ex(const void* x, int n, int l, int c, int k, int stride, const void* w, const void* bias, int act,
                           float lo, float hi, void* out, long long ldo, int lp, int padl, void* stream) {
    B200_REQUIRE(x && w && out, "conv_first_ex: null pointer argument");
    B200_REQUIRE(n >= 0 && l > 0 && lp > 0 && padl >= 0, "conv_first_ex: bad sizes n=%d l=%d lp=%d padl=%d", n, l, lp, padl);
    if (n == 0) return 0;
    B200_REQUIRE(n <= 65535, "conv_first_ex: at most 65535 chunks per call (n=%d)", n);
    return launch_conv_first_ex((const __half*)x, n, l, c, k, stride, (const __half*)w, (const __half*)bias, act, lo, hi,
                                (__half*)out, ldo, lp, padl, (cudaStream_t)stream);
}

int b200_depthwise_conv_fwd(const void* x, long long ldx, const void* w, void* y, long long ldy, int n, int t, int c, int k,
                            void* stream) {
    B200_REQUIRE(x && w && y, "depthwise: null pointer argument");
    B200_REQUIRE(n >= 0 && t >= 0, "depthwise: bad sizes n=%d t=%d", n, t);
    if (n == 0 || t == 0) return 0;
    B200_REQUIRE(n <= 65535, "depthwise: at most 65535 chunks per call (n=%d)", n);
    return launch_depthwise((const __half*)x, ldx, (const __half*)w, (__half*)y, ldy, n, t, c, k, (cudaStream_t)stream);
}

int b200_ctc_head_fwd(const void* x, long long m, int f, const void* w, const void* bias, void* logp, void* labels, void* probs,
                      void* stream) {
    B200_REQUIRE(x && w && labels && probs, "ctc_head: null pointer argument");
    B200_REQUIRE(m >= 0, "ctc_head: bad row count %lld", m);
    if (m == 0) return 0;
    return launch_ctc_head((const __half*)x, m, f, (const __half*)w, (const __half*)bias, (__half*)logp, (uint8_t*)labels,
                           (float*)probs, (cudaStream_t)stream);
}

size_t b200_sw_align_workspace_bytes(int n_pairs, int max_ref_len) { return sw_align_workspace_bytes(n_pairs, max_ref_len); }

int b200_sw_align(const void* query, const long long* query_off, const int* query_len, const void* ref, const long long* ref_off,
                  const int* ref_len, int n_pairs, void* workspace, void* out, void* stream) {
    return launch_sw_align((const uint8_t*)query, query_off, query_len, (const uint8_t*)ref, ref_off, ref_len, n_pairs,
                           workspace, (int*)out, (cudaStream_t)stream);
}

size_t b200_pair_align_trace_bytes(int mode, int query_len, int ref_len, int band) {
    return pair_align_trace_bytes(mode, query_len, ref_len, band);
}

size_t b200_pair_align_workspace_bytes(int mode, int n_pairs, const int* query_len, const int* ref_len, const int* band,
                                       int traceback) {
    return pair_align_workspace_bytes(mode, n_pairs, query_len, ref_len, band, traceback);
}

int b200_pair_align(int mode, const void* query, const long long* query_off, const int* query_len, const void* ref,
                    const long long* ref_off, const int* ref_len, const int* band, int n_pairs, int traceback, void* workspace,
                    void* ops, const long long* ops_off, void* out, void* stream) {
    return launch_pair_align(mode, (const uint8_t*)query, query_off, query_len, (const uint8_t*)ref, ref_off, ref_len, band,
                             n_pairs, traceback, workspace, (uint8_t*)ops, ops_off, (int*)out, (cudaStream_t)stream);
}

int b200_attention_fwd(void* qkv, const void* cos_sin, void* out, int n, int t, int heads, int head_dim, int wl,
                       int wr, void* stream) {
    B200_REQUIRE(qkv && cos_sin && out, "attention: null pointer argument");
    B200_REQUIRE(n >= 0 && t >= 0 && heads > 0, "attention: bad sizes n=%d t=%d heads=%d", n, t, heads);
    if (n == 0 || t == 0) return 0;
    return launch_attention((__half*)qkv, (const __half*)cos_sin, (__half*)out, n, t, heads, head_dim, wl, wr,
                            (cudaStream_t)stream);
}

int b200_rmsnorm_residual_fwd(const void* a, const void* x, const void* w, float alpha, float eps, void* out,
                              long long m, int d, void* stream) {
    B200_REQUIRE(a && x && w && out, "rmsnorm: null pointer argument");
    if (m <= 0) return 0;
    return launch_rmsnorm_residual((const __half*)a, (const __half*)x, (const __half*)w, alpha, eps, (__half*)out, m, d,
                                   (cudaStream_t)stream);
}

int b200_swiglu_fwd(const void* h, void* out, long long m, int f, void* stream) {
    B200_REQUIRE(h && out, "swiglu: null pointer argument");
    if (m <= 0) return 0;
    return launch_swiglu((const __half*)h, (__half*)out, m, f, (cudaStream_t)stream);
}

int b200_lstm_cluster_size(int hidden) { return lstm_rec_cluster_size(hidden); }

int b200_lstm_rec_fwd(const void* gx, const void* whh, void* y, int t, int n, int hidden, int reverse,
                      void* stream) {
    B200_REQUIRE(gx && whh && y, "lstm_rec: null pointer argument");
    B200_REQUIRE(t >= 0 && n >= 0, "lstm_rec: bad sizes t=%d n=%d", t, n);
    if (t == 0 || n == 0) return 0;
    return launch_lstm_rec((const __half*)gx, (const __half*)whh, (__half*)y, t, n, hidden, reverse,
                           (cudaStream_t)stream);
}

int b200_lstm_tile_chunks(int hidden) { return lstm_rec_tile_chunks(hidden); }

int b200_lstm_tile_cluster(int hidden) { return lstm_rec_tile_cluster(hidden); }

size_t b200_lstm_rec_tile_workspace_bytes(int n) { return lstm_rec_tile_workspace_bytes(n); }

int b200_lstm_rec_tile_fwd(const void* gx, const void* whh, void* y, void* workspace, int t, int n, int hidden,
                           int reverse, void* stream) {
    B200_REQUIRE(gx && whh && y && workspace, "lstm_rec_tile: null pointer argument");
    B200_REQUIRE(t >= 0 && n >= 0, "lstm_rec_tile: bad sizes t=%d n=%d", t, n);
    if (t == 0 || n == 0) return 0;
    return launch_lstm_rec_tile((const __half*)gx, (const __half*)whh, (__half*)y, workspace, t, n, hidden, reverse,
                               (cudaStream_t)stream);
}

int b200_lstm_fused_tile_fwd(const void* x, const void* wih, const void* bias, const void* whh, void* y, void* workspace,
                             int t, int n, int hidden, int reverse, void* stream) {
    B200_REQUIRE(x && wih && bias && whh && y && workspace, "lstm_fused_tile: null pointer argument");
    B200_REQUIRE(t >= 0 && n >= 0, "lstm_fused_tile: bad sizes t=%d n=%d", t, n);
    if (t == 0 || n == 0) return 0;
    return launch_lstm_fused_tile((const __half*)x, (const __half*)wih, (const __half*)bias, (const __half*)whh, (__half*)y,
                                  workspace, t, n, hidden, reverse, (cudaStream_t)stream);
}

int b200_lstm_wide_ctas(int hidden) { return lstm_rec_wide_ctas(hidden); }

int b200_lstm_wide_max_chunks(int hidden) { return lstm_rec_wide_max_chunks(hidden); }

int b200_lstm_wide_resident(int hidden) { return lstm_rec_wide_resident(hidden); }

size_t b200_lstm_rec_wide_workspace_bytes(int n, int hidden) { return lstm_rec_wide_workspace_bytes(n, hidden); }

size_t b200_lstm_rec_wide_status_offset(int n, int hidden) { return lstm_rec_wide_status_offset(n, hidden); }

int b200_lstm_rec_wide_fwd(const void* gx, const void* whh, void* y, void* workspace, int t, int n, int hidden, int reverse,
                           void* stream) {
    B200_REQUIRE(gx && whh && y && workspace, "lstm_rec_wide: null pointer argument");
    B200_REQUIRE(t >= 0 && n >= 0, "lstm_rec_wide: bad sizes t=%d n=%d", t, n);
    if (t == 0 || n == 0) return 0;
    return launch_lstm_rec_wide((const __half*)gx, (const __half*)whh, (__half*)y, workspace, t, n, hidden, reverse,
                                (cudaStream_t)stream);
}

size_t b200_crf_decode_workspace_bytes(int n, int t, int state_len) {
    return crf_decode_workspace_bytes(n, t, state_len);
}

int b200_crf_decode(const void* scores, int n, int t, int state_len, float blank_score, float qscale, float qbias,
                    void* workspace, void* moves, void* sequence, void* qstring, void* stream) {
    B200_REQUIRE(n >= 0 && t >= 0, "crf_decode: bad sizes n=%d t=%d", n, t);
    if (n == 0 || t == 0) return 0;
    B200_REQUIRE(scores && workspace && moves && sequence && qstring, "crf_decode: null pointer argument");
    return launch_crf_decode((const __half*)scores, n, t, state_len, blank_score, qscale, qbias, workspace,
                             (uint8_t*)moves, (uint8_t*)sequence, (uint8_t*)qstring, (cudaStream_t)stream);
}

int b200_crf_decode_lb(const void* scores, int n, int t, int state_len, float qscale, float qbias, void* workspace, void* moves,
                       void* sequence, void* qstring, void* stream) {
    B200_REQUIRE(n >= 0 && t >= 0, "crf_decode_lb: bad sizes n=%d t=%d", n, t);
    if (n == 0 || t == 0) return 0;
    B200_REQUIRE(scores && workspace && moves && sequence && qstring, "crf_decode_lb: null pointer argument");
    B200_REQUIRE(((uintptr_t)scores & 15) == 0, "crf_decode_lb: scores must be 16-byte aligned");
    return launch_crf_decode_lb((const __half*)scores, n, t, state_len, qscale, qbias, workspace, (uint8_t*)moves,
                                (uint8_t*)sequence, (uint8_t*)qstring, (cudaStream_t)stream);
}

int b200_chunk_count(long long length, int chunksize, int overlap) {
    if (length <= 0 || chunksize <= 0 || overlap < 0 || overlap >= chunksize) return 0;
    return chunk_count(length, chunksize, overlap);
}

int b200_chunk_signal(const void* signal, int signal_is_f32, long long length, int chunksize, int overlap, void* out,
                      long long row_stride, void* stream) {
    B200_REQUIRE(signal && out, "chunk_signal: null pointer argument");
    return launch_chunk_signal(signal, signal_is_f32, length, chunksize, overlap, (__half*)out, row_stride, (cudaStream_t)stream);
}

int b200_stream_create(void** stream_out) {
    B200_REQUIRE(stream_out != nullptr, "stream_create: null pointer argument");
    cudaStream_t st = nullptr;
    B200_CHECK_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    *stream_out = (void*)st;
    return 0;
}

int b200_quantize_i8(const void* x, void* out, long long n, float scale, void* stream) {
    B200_REQUIRE(n >= 0, "quantize_i8: bad element count %lld", n);
    if (n == 0) return 0;   // an empty tensor may have a null data pointer
    B200_REQUIRE(x && out, "quantize_i8: null pointer argument");
    return launch_quantize_i8((const __half*)x, (int8_t*)out, n, scale, (cudaStream_t)stream);
}

int b200_gemm_i8_fwd(const void* a, long long lda, const void* b, const void* col_scale, const void* bias, void* c,
                     long long ldc, int m, int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                     long long stride_inner, long long stride_outer, int group, long long stride_group, int cb_width,
                     int cb_rows, int max_ctas, void* stream) {
    B200_REQUIRE(a && b && c && col_scale, "gemm_i8: null pointer argument");
    B200_REQUIRE(m >= 0 && n > 0 && k > 0 && rows_inner > 0 && group >= 0 && n % 8 == 0 && ldc % 8 == 0,
                 "gemm_i8: bad sizes m=%d n=%d k=%d", m, n, k);
    B200_REQUIRE(cb_width >= 0 && cb_rows >= 0 && cb_width % 32 == 0, "gemm_i8: column blocks must be multiples of 32 columns");
    if (m == 0) return 0;
    GemmEpilogue ep;
    ep.bias = (const __half*)bias;
    ep.act = act;
    ep.lo = lo;
    ep.hi = hi;
    ep.map = RowMap{rows_inner, valid_inner, stride_inner, stride_outer, group, stride_group};
    ep.cb_width = cb_width;
    ep.cb_rows = cb_rows;
    return launch_gemm_i8((const int8_t*)a, lda, (const int8_t*)b, (const float*)col_scale, (__half*)c, ldc, m, n, k, ep, max_ctas,
                          (cudaStream_t)stream);
}

int b200_lstm_crf_fwd(const b200_lstm_crf_plan* plan, const void* x, void* scores, void* stream) {
    return launch_lstm_crf_fwd(plan, (const __half*)x, (__half*)scores, (cudaStream_t)stream);
}

int b200_lstm_crf_lstm_fwd(const b200_lstm_crf_plan* plan, int first, int count, void* stream) {
    B200_REQUIRE(plan != nullptr, "lstm_crf_lstm: null plan");
    return launch_lstm_stack(plan, first, count, (cudaStream_t)stream);
}

int b200_crf_beam_search(const void* scores, int n, int t, int state_len, float blank_score, int beam_width, float beam_cut,
                         float qscale, float qbias, void* workspace, void* moves, void* sequence, void* qstring, void* stream) {
    B200_REQUIRE(n >= 0 && t >= 0, "beam_search: bad sizes n=%d t=%d", n, t);
    if (n == 0 || t == 0) return 0;
    B200_REQUIRE(scores && workspace && moves && sequence && qstring, "beam_search: null pointer argument");
    return launch_crf_beam_search((const __half*)scores, n, t, state_len, blank_score, beam_width, beam_cut, qscale, qbias,
                                  workspace, (uint8_t*)moves, (uint8_t*)sequence, (uint8_t*)qstring, (cudaStream_t)stream);
}

size_t b200_ctc_crf_sparse_workspace_bytes(int n, int t, int state_len, int semiring) {
    if (n < 0 || t < 0 || state_len < 1 || state_len > 5) return 0;
    return ctc_crf_sparse_workspace_bytes(n, t, state_len, semiring);
}

#define CTC_CRF_CHECK_SPARSE(what)                                                                                      \
    B200_REQUIRE(n >= 0 && t >= 1, what ": bad sizes n=%d t=%d", n, t);                                                 \
    B200_REQUIRE(semiring == B200_SEMIRING_LOG || semiring == B200_SEMIRING_MAX, what ": unknown semiring %d", semiring); \
    B200_REQUIRE(scores && ((uintptr_t)scores & 15) == 0, what ": scores must be a 16-byte aligned device pointer")

int b200_ctc_crf_sparse_fwd(const void* scores, int t, int n, int state_len, int semiring, void* logz, void* alpha,
                            void* workspace, void* stream) {
    CTC_CRF_CHECK_SPARSE("ctc_crf_sparse_fwd");
    B200_REQUIRE(logz, "ctc_crf_sparse_fwd: null logz");
    if (n == 0) return 0;
    return launch_ctc_crf_sparse_fwd((const float*)scores, t, n, state_len, semiring, (float*)logz, (float*)alpha, workspace,
                                     (cudaStream_t)stream);
}

int b200_ctc_crf_sparse_bwd(const void* scores, int t, int n, int state_len, int semiring, void* beta, void* stream) {
    CTC_CRF_CHECK_SPARSE("ctc_crf_sparse_bwd");
    B200_REQUIRE(beta, "ctc_crf_sparse_bwd: null beta");
    if (n == 0) return 0;
    return launch_ctc_crf_sparse_bwd((const float*)scores, t, n, state_len, semiring, (float*)beta, (cudaStream_t)stream);
}

int b200_ctc_crf_sparse_grad(const void* scores, int t, int n, int state_len, int semiring, const void* g, void* workspace,
                             void* grad, void* stream) {
    CTC_CRF_CHECK_SPARSE("ctc_crf_sparse_grad");
    B200_REQUIRE(g && workspace && grad, "ctc_crf_sparse_grad: null pointer argument");
    if (n == 0) return 0;
    return launch_ctc_crf_sparse_grad((const float*)scores, t, n, state_len, semiring, (const float*)g, workspace,
                                      (float*)grad, (cudaStream_t)stream);
}

int b200_ctc_crf_target_max_states(void) { return ctc_crf_target_max_states(); }

size_t b200_ctc_crf_target_workspace_bytes(int n, int t, int l, int semiring) {
    if (n < 0 || t < 0 || l < 1) return 0;
    return ctc_crf_target_workspace_bytes(n, t, l, semiring);
}

#define CTC_CRF_CHECK_TARGET(what)                                                                                      \
    B200_REQUIRE(n >= 0 && t >= 1 && l >= 1 && l <= ctc_crf_target_max_states(),                                        \
                 what ": bad sizes n=%d t=%d l=%d (1 <= l <= %d)", n, t, l, ctc_crf_target_max_states());              \
    B200_REQUIRE(semiring == B200_SEMIRING_LOG || semiring == B200_SEMIRING_MAX, what ": unknown semiring %d", semiring); \
    B200_REQUIRE(stay && lengths && (move || l == 1), what ": null pointer argument")

int b200_ctc_crf_target_fwd(const void* stay, const void* move, const void* lengths, int t, int n, int l, int semiring,
                            void* logz, void* workspace, void* stream) {
    CTC_CRF_CHECK_TARGET("ctc_crf_target_fwd");
    B200_REQUIRE(logz, "ctc_crf_target_fwd: null logz");
    if (n == 0) return 0;
    return launch_ctc_crf_target_fwd((const float*)stay, (const float*)move, (const int*)lengths, t, n, l, semiring,
                                     (float*)logz, workspace, (cudaStream_t)stream);
}

int b200_ctc_crf_target_grad(const void* stay, const void* move, const void* lengths, int t, int n, int l, int semiring,
                             const void* g, void* workspace, void* dstay, void* dmove, void* stream) {
    CTC_CRF_CHECK_TARGET("ctc_crf_target_grad");
    B200_REQUIRE(g && workspace && dstay && (dmove || l == 1), "ctc_crf_target_grad: null pointer argument");
    if (n == 0) return 0;
    return launch_ctc_crf_target_grad((const float*)stay, (const float*)move, (const int*)lengths, t, n, l, semiring,
                                      (const float*)g, workspace, (float*)dstay, (float*)dmove, (cudaStream_t)stream);
}

size_t b200_ctc_beam_workspace_bytes(int n_reads, long long total_frames, int beam_width) {
    return ctc_beam_workspace_bytes(n_reads, total_frames, beam_width);
}

int b200_ctc_beam_search(const void* logp, const long long* frame_off, const int* frame_len, int n_reads, int beam_width,
                         float threshold, float qscale, float qbias, void* workspace, size_t workspace_bytes, void* sequence,
                         void* qstring, void* moves, void* stream) {
    return launch_ctc_beam_search((const __half*)logp, frame_off, frame_len, n_reads, beam_width, threshold, qscale, qbias,
                                  workspace, workspace_bytes, (uint8_t*)sequence, (uint8_t*)qstring, (uint8_t*)moves,
                                  (cudaStream_t)stream);
}

}  // extern "C"
