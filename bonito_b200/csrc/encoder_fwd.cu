// Coarse entry point of the LSTM-CRF encoder: the whole forward of one batch -- fused conv stem, strided convolution GEMM,
// n_lstm x persistent LSTM layer with its input projection fused in (in chains of tiles on the plan's chain streams),
// LinearCRFEncoder GEMM (+Clamp) -- enqueued from one C call, on caller-owned buffers in the tile layout.
// Reference span: the `encoder` Serial of a bonito.crf model (bonito/crf/model.py:150-162, bonito/nn.py:221-298,353-415),
// i.e. what `Model.use_koi` hands to koi.lstm.update_graph plus the layers around it.
#include "common.cuh"

int launch_conv_stem(const __half* x, int N, int L, int C1, int K1, const __half* w1, const __half* b1, int act1,
                     int C2, int K2, const __half* w2, const __half* b2, int act2, __half* out, int Lp, int padl,
                     float lo1, float hi1, float lo2, float hi2, cudaStream_t stream);
int launch_lstm_fused_tile(const __half* x, const __half* wih, const __half* bias, const __half* whh, __half* y,
                           void* workspace, int T, int N, int hidden, int reverse, cudaStream_t stream);
int lstm_rec_tile_chunks(int hidden);
size_t lstm_rec_tile_workspace_bytes(int N);

// LSTM layers [first, first + count) in chains of consecutive tiles, chain c on its own stream, forked from and joined back
// into `stream`.  Tile k of a layer needs only tile k of the layer before, so a chain runs its tiles through all the layers
// without waiting for the other tiles.  With two batches in flight this matters: an H100 holds 15 of the kernel's 8-CTA
// clusters, one fewer than two 8-tile layers need, and with one launch per layer the later layer's last cluster waited for
// the whole other layer (hac step 36.5 ms; 2 chains 34.0 ms, 4 chains 32.3 ms, 8 chains 32.4 ms on an H100 80GB HBM3 at
// 700 W).  Each launch computes its tiles exactly as one launch per layer does.
int launch_lstm_stack(const b200_lstm_crf_plan* p, int first, int count, cudaStream_t stream) {
    const int H = p->hidden, TB = lstm_rec_tile_chunks(H), N = p->n, T = p->t;
    const int nt = (N + TB - 1) / TB;
    B200_REQUIRE(TB > 0 && first >= 0 && count >= 0 && first + count <= p->n_lstm,
                 "lstm_crf_lstm: layers [%d, %d) of %d, hidden size %d", first, first + count, p->n_lstm, H);
    cudaStream_t st[B200_LSTM_CHAINS] = {stream};
    int chains = 1;
    while (chains < B200_LSTM_CHAINS && chains < nt && p->chain_streams[chains - 1]) {
        st[chains] = (cudaStream_t)p->chain_streams[chains - 1];
        ++chains;
    }
    cudaEvent_t ev[B200_LSTM_CHAINS];   // ev[0]: the fork; ev[c]: chain c done
    for (int c = 0; c < chains && chains > 1; ++c) B200_CHECK_CUDA(cudaEventCreateWithFlags(&ev[c], cudaEventDisableTiming));
    if (chains > 1) B200_CHECK_CUDA(cudaEventRecord(ev[0], stream));
    const size_t tile_elems = (size_t)T * TB * H, tile_ws = lstm_rec_tile_workspace_bytes(TB);
    int rc = 0;
    for (int c = 0; c < chains && rc == 0; ++c) {
        const int t0 = nt * c / chains, t1 = nt * (c + 1) / chains;
        if (c > 0) B200_CHECK_CUDA(cudaStreamWaitEvent(st[c], ev[0], 0));
        for (int i = first; i < first + count && rc == 0; ++i) {
            const __half* src = (const __half*)(i % 2 ? p->yb : p->ya) + t0 * tile_elems;
            __half* dst = (__half*)(i % 2 ? p->ya : p->yb) + t0 * tile_elems;
            rc = launch_lstm_fused_tile(src, (const __half*)p->wih[i], (const __half*)p->bias[i], (const __half*)p->whh[i], dst,
                                        (unsigned char*)p->hx + t0 * tile_ws, T, min(N - t0 * TB, (t1 - t0) * TB), H,
                                        p->reverse[i], st[c]);
        }
        if (c > 0 && rc == 0) {
            B200_CHECK_CUDA(cudaEventRecord(ev[c], st[c]));
            B200_CHECK_CUDA(cudaStreamWaitEvent(stream, ev[c], 0));
        }
    }
    for (int c = 0; c < chains && chains > 1; ++c) cudaEventDestroy(ev[c]);   // released once the work using them is done
    return rc;
}

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
    rc = launch_lstm_stack(p, 0, p->n_lstm, stream);
    if (rc) return rc;
    if (p->n_lstm % 2) cur = nxt;
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
