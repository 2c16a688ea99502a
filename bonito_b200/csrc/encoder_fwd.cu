// Coarse entry point of the LSTM-CRF encoder: the whole forward of one batch -- fused conv stem, strided convolution GEMM,
// n_lstm x persistent LSTM layer with its input projection fused in, LinearCRFEncoder GEMM (+Clamp) -- enqueued on one
// stream from one C call (9 kernel launches for the hac shape), on caller-owned buffers in the tile layout.
// Reference span: the `encoder` Serial of a bonito.crf model (bonito/crf/model.py:150-162, bonito/nn.py:221-298,353-415),
// i.e. what `Model.use_koi` hands to koi.lstm.update_graph plus the layers around it.
#include "common.cuh"

int launch_conv_stem(const __half* x, int N, int L, int C1, int K1, const __half* w1, const __half* b1, int act1,
                     int C2, int K2, const __half* w2, const __half* b2, int act2, __half* out, int Lp, int padl,
                     float lo1, float hi1, float lo2, float hi2, cudaStream_t stream);
int launch_lstm_fused_tile(const __half* x, const __half* wih, const __half* bias, const __half* whh, __half* y,
                           void* workspace, int T, int N, int hidden, int reverse, cudaStream_t stream);
int lstm_rec_tile_chunks(int hidden);

int launch_lstm_crf_fwd(const b200_lstm_crf_plan* p, const __half* x, __half* scores, cudaStream_t stream) {
    B200_REQUIRE(p != nullptr && x != nullptr && scores != nullptr, "lstm_crf_fwd: null pointer argument");
    const int H = p->hidden, TB = lstm_rec_tile_chunks(H);
    B200_REQUIRE(TB > 0, "lstm_crf_fwd: hidden size %d has no tile-layout recurrent kernel", H);
    B200_REQUIRE(p->n_lstm >= 1 && p->n_lstm <= B200_MAX_LSTM_LAYERS, "lstm_crf_fwd: %d LSTM layers are not supported", p->n_lstm);
    const int N = p->n, L = p->l, T = p->t, Tp = p->tp, Lp = Tp * p->s3;
    B200_REQUIRE(N > 0 && L > 0 && T > 0 && Tp >= T, "lstm_crf_fwd: bad geometry n=%d l=%d t=%d tp=%d", N, L, T, Tp);
    // the plan carries no bounds for the convolutions: clamped activations go through the layer-by-layer entry points
    B200_REQUIRE(p->act1 != B200_ACT_SWISH_CLAMP && p->act2 != B200_ACT_SWISH_CLAMP && p->act3 != B200_ACT_SWISH_CLAMP,
                 "lstm_crf_fwd: B200_ACT_SWISH_CLAMP needs bounds the plan does not carry");
    __half* stem = (__half*)p->stem;
    __half* cur = (__half*)p->ya;
    __half* nxt = (__half*)p->yb;

    int rc = launch_conv_stem(x, N, L, p->c1, p->k1, (const __half*)p->w1, (const __half*)p->b1, p->act1, p->c2, p->k2,
                              (const __half*)p->w2, (const __half*)p->b2, p->act2, stem, Lp, p->pad3, 0.f, 0.f, 0.f, 0.f,
                              stream);
    if (rc) return rc;
    GemmEpilogue ep;
    // strided convolution: rows r = n*Tp + t are windows of k3*c2 elements, s3*c2 apart -> ya[tile n/TB][t][n%TB]
    ep.bias = (const __half*)p->b3; ep.act = p->act3; ep.lo = ep.hi = 0.f;
    ep.map = RowMap{Tp, T, (long long)TB, 1, TB, (long long)T * TB};
    ep.cb_width = ep.cb_rows = 0;
    rc = launch_gemm_tc(stem, (long long)p->s3 * p->c2, (const __half*)p->w3, cur, H, N * Tp, H, p->k3 * p->c2, ep, 0, stream);
    if (rc) return rc;
    for (int i = 0; i < p->n_lstm; ++i) {
        rc = launch_lstm_fused_tile(cur, (const __half*)p->wih[i], (const __half*)p->bias[i], (const __half*)p->whh[i], nxt,
                                    p->hx, T, N, H, p->reverse[i], stream);
        if (rc) return rc;
        __half* tmp = cur; cur = nxt; nxt = tmp;
    }
    // LinearCRFEncoder (+Clamp): rows r = (tile*T + t)*TB + i -> scores[tile*TB + i][t]; a partial last tile separately
    ep.bias = (const __half*)p->bl; ep.act = p->act_l; ep.lo = p->lo; ep.hi = p->hi;
    const int full = N / TB;
    if (full > 0) {
        ep.map = RowMap{TB, TB, (long long)T, 1, T, (long long)TB * T};
        rc = launch_gemm_tc(cur, H, (const __half*)p->wl, scores, p->n_scores, full * T * TB, p->n_scores, H, ep, 0, stream);
        if (rc) return rc;
    }
    if (N % TB) {
        ep.map = RowMap{TB, N % TB, (long long)T, 1, 0, 0};
        rc = launch_gemm_tc(cur + (size_t)full * T * TB * H, H, (const __half*)p->wl, scores + (size_t)full * TB * T * p->n_scores,
                            p->n_scores, T * TB, p->n_scores, H, ep, 0, stream);
        if (rc) return rc;
    }
    return 0;
}
