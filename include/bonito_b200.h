/*
 * bonito_b200 -- C ABI of the H100-native (sm_90a) chunked forward + decode path.
 *
 * The reference (nanoporetech/bonito) is pure Python; its native work on this path is done by
 * third-party binaries reached from these call sites, which are what each entry point replaces:
 *
 *   b200_conv_stem_fwd        torch.nn.Conv1d x2 + activations        bonito/nn.py:221-241
 *                             (_ex: + Clamp behind each, dna_r10.4.1@v4.0)
 *   b200_gemm_fwd             torch.nn.Conv1d (strided, as GEMM),     bonito/nn.py:226,283-298,59-67
 *                             torch.nn.Linear + Clamp (LinearCRFEncoder, the Linear in front of it), LSTM input projection
 *   b200_lstm_rec_fwd         koi.lstm.update_graph / torch.nn.LSTM   bonito/crf/model.py:240-246, bonito/nn.py:366-370
 *   b200_depthwise_conv_fwd   TCSConv1d.depthwise (QuartzNet CTC)      bonito/ctc/model.py:90-121
 *   b200_ctc_head_fwd         Decoder + log_softmax, greedy argmax     bonito/ctc/model.py:195-208, ctc/basecall.py:53-58
 *   b200_sw_align             parasail.sw_trace_striped_32 + CIGAR    bonito/cli/evaluate.py:37-67
 *                             counts (`evaluate`)
 *   b200_pair_align           edlib.align(task="path") and            bonito/cli/duplex.py:225-273
 *                             parasail.sg_trace_scan_32 (`duplex`)
 *   b200_crf_decode           koi.decode.beam_search call contract    bonito/crf/basecall.py:36-40
 *                             with SeqdistModel.decode_batch maths    bonito/crf/model.py:98-108,196-199
 *                             (_lb: learned blank scores, heads without blank_score, bonito/crf/model.py:150-162)
 *   b200_ctc_crf_*            koi.ctc (logZ_cu_sparse, fwd/bwd_scores_  bonito/crf/model.py:30-143
 *                             cu_sparse, logZ_cu, viterbi_alignments)
 *   b200_ctc_beam_search      fast_ctc_decode.beam_search             bonito/ctc/model.py:39-46, ctc/basecall.py:43-61
 *   b200_bgzf_compress        htslib bgzf_write, reached through      bonito/io.py:400-503
 *                             pysam AlignmentFile(..., 'wb') (BAM output)
 *
 * Conventions (SURVEY.md section 8b): every function returns 0 on success and a negative value on
 * failure, with a message available from b200_last_error().  All pointers are raw DEVICE pointers
 * owned by the caller (fp16 = IEEE binary16); the library never allocates or frees caller memory and
 * keeps no thread-local CUDA state: work is enqueued on the `stream` argument (a cudaStream_t passed
 * as void*) of the device that is current on the calling thread.  Workspace sizes come from the
 * *_workspace_bytes() queries.  Safe to call from any host thread.
 */
#ifndef BONITO_B200_H
#define BONITO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ACT_NONE 0
#define B200_ACT_SWISH 1
#define B200_ACT_TANH 2
#define B200_ACT_CLAMP 3 /* clamp(lo, hi), Clamp layer: bonito/nn.py:59-67 */
#define B200_ACT_SCALE 4 /* multiply by lo, LinearCRFEncoder.scale: bonito/nn.py:288-289 */
/* SwiGLU fused into the GEMM (wgmma path only): the n output columns are 64-wide groups [32 x y | 32 x gate] (the caller
 * interleaves the rows of fc1.weight that way) and c receives n/2 columns, c[:, 32*g + j] = gate * y / (1 + exp(-gate)) on the
 * fp16-rounded y / gate, rounded once -- GatedMlp: flash_attn/modules/mlp.py:99-136, flash_attn/ops/activations.py:107-111
 * as used by bonito/transformer/model.py:100-104.  n % 64 == 0, no bias. */
#define B200_ACT_SWIGLU 5
#define B200_ACT_TANH_SCALE 6 /* tanh, then multiply by lo: LinearCRFEncoder(activation="tanh", scale=5.0), bonito/nn.py:283-298 */
/* swish, rounded to fp16, then clamp(lo, hi): a Convolution with activation "swish" followed by a Clamp layer
 * (dna_r10.4.1@v4.0: Clamp(-0.5, 3.5) after each of the three convolutions) */
#define B200_ACT_SWISH_CLAMP 7
#define B200_ACT_RELU 8 /* max(x, 0): the QuartzNet CTC model dna_r9.4.1@v1 (bonito/ctc/model.py, [encoder] activation = "relu") */

#define B200_GEMM_AUTO 0 /* the wgmma kernel (product path) unless B200_GEMM_IMPL=mma is set in the environment */
#define B200_GEMM_TCGEN05 1 /* the wgmma kernel (the name is kept for ABI compatibility) */
#define B200_GEMM_MMA_SYNC 2 /* legacy tensor path, kept for on-device cross-checks */

/* Library version (major*10000 + minor*100 + patch). */
int b200_version(void);

/* Message of the last failure ON THE CALLING THREAD ("" if none); the buffer is thread-local and stays valid until the
 * same thread fails again. */
const char* b200_last_error(void);

/*
 * Fused conv stem: x[N][L] -> Conv1d(1->c1,k1,pad k1/2)+act1 -> Conv1d(c1->c2,k2,pad k2/2)+act2,
 * written channels-last and zero padded: out[n][padl + l][c], `lp` rows per chunk (rows outside
 * [padl, padl+L) are written as zeros).  Weights in torch layout (w1 [c1][1][k1], w2 [c2][c1][k2]),
 * biases may be NULL.  Supported shapes: (c1,k1,c2,k2) = (16,5,16,5), (4,5,16,5).
 */
int b200_conv_stem_fwd(const void* x, int n, int l, int c1, int k1, const void* w1, const void* b1, int act1,
                       int c2, int k2, const void* w2, const void* b2, int act2, void* out, int lp, int padl,
                       void* stream);
/* Same, with the bounds (lo1, hi1) / (lo2, hi2) of act1 / act2 (used by B200_ACT_SWISH_CLAMP and B200_ACT_CLAMP; the entry
 * point above passes zeros). */
int b200_conv_stem_fwd_ex(const void* x, int n, int l, int c1, int k1, const void* w1, const void* b1, int act1, float lo1,
                          float hi1, int c2, int k2, const void* w2, const void* b2, int act2, float lo2, float hi2, void* out,
                          int lp, int padl, void* stream);

/*
 * C = act(A[M,K] * B[N,K]^T + bias) in fp16 with fp32 accumulation.
 *   A: row stride `lda` elements (lda < K is allowed: overlapping rows = strided convolution windows)
 *   B: [N][K] row-major (torch Linear / packed Conv1d weight), bias[N] or NULL
 *   output row of input row r: (outer, inner) = divmod(r, rows_inner); rows with inner >= valid_inner are
 *   skipped; out_row = inner*stride_inner + outer*stride_outer; C row stride `ldc` elements.
 *   (identity mapping: rows_inner = valid_inner = M, stride_inner = 1, stride_outer = 0)
 * Requirements: K % 8 == 0, lda % 8 == 0, N % 8 == 0, ldc % 8 == 0, A/B/C 16-byte aligned.
 */
int b200_gemm_fwd(const void* a, long long lda, const void* b, const void* bias, void* c, long long ldc, int m,
                  int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                  long long stride_inner, long long stride_outer, int impl, void* stream);

/*
 * Same, with
 *   max_ctas  accepted for compatibility and ignored: the wgmma kernel is not persistent (its CTAs leave as they finish);
 *   group, stride_group  second level of the row map (group = 0: off): (outer2, outer1) = divmod(outer, group),
 *             out_row = inner*stride_inner + outer1*stride_outer + outer2*stride_group -- e.g. chunk n -> (tile n/48, n%48);
 *   cb_width, cb_rows  column blocks (cb_width = 0: off; multiple of 32): output column c of mapped row R is written to
 *             row R + (c / cb_width) * cb_rows, column c % cb_width.  With ldc = cb_width this lays the LSTM input
 *             projection out as [t][cluster rank][chunk][cb_width], one contiguous block per recurrent CTA and step.
 */
int b200_gemm_fwd_ex(const void* a, long long lda, const void* b, const void* bias, void* c, long long ldc, int m,
                     int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                     long long stride_inner, long long stride_outer, int group, long long stride_group, int cb_width,
                     int cb_rows, int impl, int max_ctas, void* stream);

/*
 * Cluster size the packed LSTM operands must be laid out for (0: hidden size unsupported).
 * Supported hidden sizes: 96, 128, 256, 384.
 */
int b200_lstm_cluster_size(int hidden);

/*
 * Recurrent part of one unidirectional LSTM layer over all T steps (h0 = c0 = 0):
 *   gx  [T][N][4H]  input projection x_t W_ih^T + b_ih + b_hh, columns permuted to
 *                   [cluster rank][unit/8 block][unit%8][gate i,f,g,o]
 *   whh [4H][H]     recurrent weights, rows permuted to [cluster rank][unit/8 block][gate][unit%8]
 *   y   [T][N][H]   h_t in natural unit order
 * reverse != 0 runs t = T-1..0 (the reference flips the sequence instead: bonito/nn.py:366-370).
 * Every supported size runs the mma.sync kernel (W_hh resident in shared memory, h exchanged through L2); the hot path of
 * hidden = 384 is the tile-layout kernel below.
 */
int b200_lstm_rec_fwd(const void* gx, const void* whh, void* y, int t, int n, int hidden, int reverse,
                      void* stream);

/*
 * Tile layout of the H = 384 recurrent kernel (clusters of 8 CTAs x 48 hidden units, W_hh slice resident in shared memory,
 * wgmma on 64-chunk tiles, h all-gather as multicast bulk copies through L2).
 *   b200_lstm_tile_chunks(hidden)   chunks per tile (64 for hidden = 384; 0 = this hidden size has no tile kernel)
 *   b200_lstm_tile_cluster(hidden)  CTAs per cluster = column blocks of gx (8)
 *   gx  [tiles][T][8][64][192]  columns of cluster rank r: [unit - 48r][gate i,f,g,o]  (b200_gemm_fwd_ex with
 *                               rows (t, chunk), cb_width = 192, cb_rows = 64, ldc = 192)
 *   whh [4H][H]                 as for b200_lstm_rec_fwd
 *   y   [tiles][T][64][H]       h_t in natural unit order; rows of chunks >= n are not written
 *   workspace                   b200_lstm_rec_tile_workspace_bytes(n) bytes (96 KB per tile): staging of the h all-gather;
 *                               contents irrelevant, but launches that may run concurrently need distinct workspaces
 * tiles = ceil(n / 64); one launch runs all of them (one cluster each).
 */
int b200_lstm_tile_chunks(int hidden);
int b200_lstm_tile_cluster(int hidden);
size_t b200_lstm_rec_tile_workspace_bytes(int n);
int b200_lstm_rec_tile_fwd(const void* gx, const void* whh, void* y, void* workspace, int t, int n, int hidden,
                           int reverse, void* stream);

/*
 * One whole fp16 LSTM layer of hidden = 384 in the tile layout, input projection included (the hot path of the hac model):
 * the same clusters, tiles and h all-gather as b200_lstm_rec_tile_fwd, with x_t W_ih^T + b computed inside the recurrence
 * (W_ih slice resident in shared memory, x_t loaded by TMA), so no gate pre-activations go through HBM.  The results are
 * bit-identical to b200_gemm_fwd_ex (wih, bias) into gx followed by b200_lstm_rec_tile_fwd.
 *   x    [tiles][T][64][H]  layer input (rows of chunks >= n are read and their results dropped: keep them finite)
 *   wih  [4H][H], bias [4H] rows in gx column order [unit][gate i,f,g,o];  whh [4H][H] as for b200_lstm_rec_fwd
 *   y    [tiles][T][64][H]  h_t in natural unit order; rows of chunks >= n are not written
 *   workspace               b200_lstm_rec_tile_workspace_bytes(n) bytes, as for b200_lstm_rec_tile_fwd
 */
int b200_lstm_fused_tile_fwd(const void* x, const void* wih, const void* bias, const void* whh, void* y, void* workspace,
                             int t, int n, int hidden, int reverse, void* stream);

/*
 * Wide recurrent kernel, hidden = 768 and 1024 (dna_r9.4.1@v3.1, dna_r10.4.1@v4.3): W_hh is spread over G = hidden / 8 CTAs
 * (8 units = 32 gate columns each, slice resident in shared memory), one cooperative launch per layer, wgmma on 64-chunk
 * tiles, h exchanged through L2 with a grid-wide barrier every step.  b200_lstm_cluster_size() keeps returning 0 for these
 * widths: it describes the generic kernel.
 *   b200_lstm_wide_ctas(hidden)        G (96 / 128), 0 = this hidden size has no wide kernel
 *   b200_lstm_wide_max_chunks(hidden)  largest n one launch accepts (2560)
 *   b200_lstm_wide_resident(hidden)    CTAs of the kernel that can be resident at once on the current device (negative on
 *                                      error); the grid only launches if this is >= G
 *   gx  [T][G][n][32]   columns of CTA g: [unit - 8g][gate i,f,g,o]  (b200_gemm_fwd_ex with W_ih / bias in [unit][gate]
 *                       row order, rows (t, chunk): rows_inner = n, stride_inner = 1, stride_outer = G*n, cb_width = 32,
 *                       cb_rows = n, ldc = 32)
 *   whh [4H][H]         as for b200_lstm_rec_fwd
 *   y   [T][n][H]       h_t in natural unit order
 *   workspace           b200_lstm_rec_wide_workspace_bytes(n, hidden) bytes: h exchange buffer, barrier counter and status
 *                       word (reset on the stream by every launch); launches that may run concurrently need distinct
 *                       workspaces
 * Status: the uint32 at byte offset b200_lstm_rec_wide_status_offset(n, hidden) of the workspace is 0 after a launch that
 * completed, non-zero if the CTAs stopped waiting for each other (a bounded wait expired) and y is not valid.
 */
int b200_lstm_wide_ctas(int hidden);
int b200_lstm_wide_max_chunks(int hidden);
int b200_lstm_wide_resident(int hidden);
size_t b200_lstm_rec_wide_workspace_bytes(int n, int hidden);
size_t b200_lstm_rec_wide_status_offset(int n, int hidden);
int b200_lstm_rec_wide_fwd(const void* gx, const void* whh, void* y, void* workspace, int t, int n, int hidden, int reverse,
                           void* stream);

/*
 * ---- transformer (sup) path: bonito/transformer/model.py ----
 *
 * First convolution of a conv stack: x[N][L] -> Conv1d(1->c, k, pad k/2) + act, channels-last with zero halo:
 * out[n][padl + l][c], `lp` rows per chunk.  The following convolutions run as b200_gemm_fwd over overlapping rows.
 */
int b200_conv_first_fwd(const void* x, int n, int l, int c, int k, const void* w, const void* bias, int act, void* out,
                        int lp, int padl, void* stream);

/*
 * Same for strided convolutions and wider outputs (the C1 block of the QuartzNet CTC models: 1 -> 256 k33 s3, 1 -> 344 k9 s3,
 * BatchNorm folded into w / bias): T = (l - 1) / stride + 1 output frames (padding k/2), frame t of chunk n written to row
 * n*lp + padl + t of `out` with row pitch `ldo` elements (so it can fill a column range of a wider buffer); the other rows
 * of [n*lp, n*lp + lp) get zeros in the c columns.  lo / hi: bounds of B200_ACT_CLAMP / B200_ACT_SWISH_CLAMP.
 * c % 8 == 0, c <= 512, odd k <= 33, 1 <= stride <= 8, ldo % 8 == 0, out 16-byte aligned.
 */
int b200_conv_first_fwd_ex(const void* x, int n, int l, int c, int k, int stride, const void* w, const void* bias, int act,
                           float lo, float hi, void* out, long long ldo, int lp, int padl, void* stream);

/*
 * ---- QuartzNet CTC path: bonito/ctc/model.py ----
 *
 * Depthwise Conv1d (groups = channels, stride 1, padding k/2, no bias) on channels-last fp16 rows:
 *   y[(n*t + i)*ldy + ch] = sum_j w[ch][j] * x[(n*t + i + j - k/2)*ldx + ch],  frames outside [0, t) of chunk n read as zero
 * w [c][1][k] fp16 (torch layout).  fp32 accumulation, one rounding to fp16.  Supported: 256 <= c <= 512, c % 8 == 0,
 * k in {5, 9, 31, 33, 39, 51, 63, 67, 75, 87, 115, 123}; ldx, ldy multiples of 8 and >= c, x 16-byte aligned.
 */
int b200_depthwise_conv_fwd(const void* x, long long ldx, const void* w, void* y, long long ldy, int n, int t, int c, int k,
                            void* stream);

/*
 * CTC head + per-frame greedy step, for m rows of f features (x [m][f] fp16, f % 8 == 0, f <= 2048, 16-byte aligned):
 *   logits = fp16(x w^T + bias)      w [5][f], bias [5] (may be NULL)
 *   logp   = fp16(log_softmax(logits)) computed in fp32, written to logp [m][5] unless logp is NULL
 *   labels [m] uint8 = argmax of logp (equal values: the highest index wins), probs [m] fp32 = exp(logp[label])
 */
int b200_ctc_head_fwd(const void* x, long long m, int f, const void* w, const void* bias, void* logp, void* labels, void* probs,
                      void* stream);

/*
 * Batched Smith-Waterman local alignment with affine gaps (match +5, mismatch -4, gap open 8, extend 4; the tie rules are
 * in bonito_b200/csrc/align.cu), for n_pairs pairs (query p, reference p) of ASCII A/C/G/T bytes.  `query` / `ref` are
 * packed DEVICE byte buffers; pair p is query[query_off[p] .. + query_len[p]) against ref[ref_off[p] .. + ref_len[p]).
 * Unlike the rest of this ABI, query_off / ref_off (int64) and query_len / ref_len (int32) are HOST arrays: the lengths
 * are checked on the host (each in [0, 65535], else -2) and the four arrays are copied into the head of `workspace` on
 * `stream`, so pinned arrays must stay unchanged until the stream has passed this call.  `workspace`: DEVICE memory of
 * b200_sw_align_workspace_bytes(n_pairs, max_ref_len) bytes with max_ref_len >= every ref_len[p].
 * out: int32 [n_pairs][7] = score, end_query, end_ref (0-based, inclusive), n_eq, n_x, n_ins, n_del of the traced
 * alignment; a pair whose best score is 0 gives 0, -1, -1, 0, 0, 0, 0.  n_pairs == 0 is a no-op.
 */
size_t b200_sw_align_workspace_bytes(int n_pairs, int max_ref_len);
int b200_sw_align(const void* query, const long long* query_off, const int* query_len, const void* ref, const long long* ref_off,
                  const int* ref_len, int n_pairs, void* workspace, void* out, void* stream);

/*
 * Batched pairwise alignment with a traceback, for `duplex` (the reference aligns with edlib.align(task="path") and
 * parasail.sg_trace_scan_32; the scoring, band and tie rules here are this library's, in bonito_b200/csrc/pair_align.cu):
 *   B200_PAIR_GLOBAL_EDIT        unit-cost global alignment restricted to the diagonals
 *                                [min(0, n-m) - band[p], max(0, n-m) + band[p]]; the result is the unbanded optimum
 *                                whenever the returned distance is <= band[p] (or band[p] >= max(m, n))
 *   B200_PAIR_SEMIGLOBAL_AFFINE  match +5, mismatch -4, gap 10 + 2 (g - 1), free end gaps, full matrix
 * Pair p is query[query_off[p] .. + query_len[p]) (rows, 'I' consumes it) against ref[ref_off[p] .. + ref_len[p])
 * (columns, 'D' consumes it); `query` / `ref` are DEVICE byte buffers (equal bytes match).  As for b200_sw_align the
 * per-pair arrays query_off, query_len, ref_off, ref_len, band (int32, GLOBAL_EDIT only, >= 0; values above max(m, n) act
 * as max(m, n)) and ops_off (int64) are HOST arrays, checked on the host (lengths in [0, 2^28], else -2) and copied into
 * the head of `workspace`.  workspace: DEVICE memory of b200_pair_align_workspace_bytes() bytes for the same arguments;
 * b200_pair_align_trace_bytes() is the share of one pair (its traceback bits).
 * traceback == 0 (GLOBAL_EDIT only): out[p][0] = the banded distance, nothing else is written and no trace bytes are needed.
 * traceback != 0: out int32 [n_pairs][2] = score (distance / affine score), n_ops; the ops, one byte each of '=', 'X',
 * 'I', 'D' in forward order, are the LAST n_ops bytes of the slot ops[ops_off[p] .. + query_len[p] + ref_len[p]) (DEVICE).
 */
#define B200_PAIR_GLOBAL_EDIT 0
#define B200_PAIR_SEMIGLOBAL_AFFINE 1
size_t b200_pair_align_trace_bytes(int mode, int query_len, int ref_len, int band);
size_t b200_pair_align_workspace_bytes(int mode, int n_pairs, const int* query_len, const int* ref_len, const int* band,
                                       int traceback);
int b200_pair_align(int mode, const void* query, const long long* query_off, const int* query_len, const void* ref,
                    const long long* ref_off, const int* ref_len, const int* band, int n_pairs, int traceback, void* workspace,
                    void* ops, const long long* ops_off, void* out, void* stream);

/*
 * Rotary embedding (NeoX half rotation, cos_sin [T][64] fp16 = cos[32] | sin[32] per position) + windowed softmax
 * attention, non-causal: key j is visible to query i iff i - wl <= j <= i + wr (negative = unlimited).
 * qkv [N][T][3][heads][64] fp16 (packed projection, bonito/transformer/model.py:71) -> out [N][T][heads*64].
 * The q and k parts of `qkv` are rotated IN PLACE (as flash-attn's RotaryEmbedding does, transformer/model.py:73).
 */
int b200_attention_fwd(void* qkv, const void* cos_sin, void* out, int n, int t, int heads, int head_dim, int wl,
                       int wr, void* stream);

/* out[r] = rmsnorm(a[r] + fp16(alpha * x[r]), eps) * w   for m rows of d elements (DeepNorm post-norm residual). */
int b200_rmsnorm_residual_fwd(const void* a, const void* x, const void* w, float alpha, float eps, void* out,
                              long long m, int d, void* stream);

/* h [m][2f] = (y | gate) -> out [m][f] = gate * y / (1 + exp(-gate))   (GatedMlp with SiLU). */
int b200_swiglu_fwd(const void* h, void* out, long long m, int f, void* stream);

/* Bytes of scratch b200_crf_decode needs for n chunks of t frames. */
size_t b200_crf_decode_workspace_bytes(int n, int t, int state_len);

/*
 * Posterior + Viterbi decode of CRF scores.
 *   scores [N][T][4^(state_len+1)] fp16, no blank column (index = state*4 + dropped_base);
 *   blank_score: fixed stay score (reference LinearCRFEncoder.blank_score / beam_search default 2.0)
 *   moves/sequence/qstring: [N][T] bytes; sequence/qstring hold an ASCII char on move frames and 0
 *   elsewhere, so `to_str` = bytes of the non-zero entries (bonito/crf/basecall.py:50-54);
 *   quality = phred of the posterior move mass of the emitted base, q = -10 log10(max(1-p,1e-4))*qscale+qbias.
 */
int b200_crf_decode(const void* scores, int n, int t, int state_len, float blank_score, float qscale, float qbias,
                    void* workspace, void* moves, void* sequence, void* qstring, void* stream);

/*
 * The same decode for heads with LEARNED blank scores (LinearCRFEncoder without blank_score, e.g. dna_r9.4.1@v3):
 *   scores [N][T][5 * 4^state_len] fp16, 16-byte aligned, in the CTC_CRF layout [state][stay, move 0..3]
 *   (bonito/crf/model.py:37-42): the stay edge of state s at frame t scores scores[t][s*5], its in-edge 1+j scores[t][s*5+1+j].
 * Same passes, arithmetic, tie-breaks, outputs and quality rule as b200_crf_decode; the workspace is the same size, so
 * b200_crf_decode_workspace_bytes(n, t, state_len) covers it.
 */
int b200_crf_decode_lb(const void* scores, int n, int t, int state_len, float qscale, float qbias, void* workspace, void* moves,
                       void* sequence, void* qstring, void* stream);

/*
 * ---- chunk() on the device (reference: bonito.util.chunk, bonito/util.py:142-161) ----
 * b200_chunk_count: number of chunks of a read of `length` samples (0 for an invalid geometry).
 * b200_chunk_signal: signal [length] (fp16, or fp32 when signal_is_f32) -> out [b200_chunk_count][chunksize] fp16, rows
 *   `row_stride` elements apart: reads shorter than a chunk are tiled, otherwise windows every chunksize - overlap samples from
 *   stub = (length - overlap) % (chunksize - overlap), preceded by signal[:chunksize] when stub > 0.
 */
int b200_chunk_count(long long length, int chunksize, int overlap);
int b200_chunk_signal(const void* signal, int signal_is_f32, long long length, int chunksize, int overlap, void* out,
                      long long row_stride, void* stream);

/*
 * b200_stream_create: a non-blocking CUDA stream on the current device, for the lifetime of the process (host frameworks
 * that hand out pooled streams -- torch: 32 per device, round-robin -- cannot promise that two streams are distinct; the
 * pipelined host loop needs its per-batch and copy streams to be).
 */
int b200_stream_create(void** stream_out);

/*
 * ---- INT8 input projection (--quantize; reference: koi's int8 LSTM path, bonito/crf/model.py:245, cli/basecaller.py:186-189) ----
 * b200_quantize_i8: out[i] = clamp(rint(x[i] * scale), -127, 127), fp16 -> int8, n a multiple of 8.
 * b200_gemm_i8_fwd: C = act(col_scale[j] * sum_k A_i8[i][k] B_i8[j][k] + bias[j]) -- int8 operands (lda in bytes), s32
 *   accumulation on the int8 tensor cores (wgmma s8), per-column float scale (weight scale / activation scale), fp16 bias /
 *   output, the same row / column-block maps as b200_gemm_fwd_ex.  K % 16 == 0, N % 8 == 0.
 */
int b200_quantize_i8(const void* x, void* out, long long n, float scale, void* stream);
int b200_gemm_i8_fwd(const void* a, long long lda, const void* b, const void* col_scale, const void* bias, void* c,
                     long long ldc, int m, int n, int k, int act, float lo, float hi, int rows_inner, int valid_inner,
                     long long stride_inner, long long stride_outer, int group, long long stride_group, int cb_width,
                     int cb_rows, int max_ctas, void* stream);

/*
 * ---- coarse entry point: the whole LSTM-CRF encoder forward of one batch from one call ----
 * conv stem -> strided convolution (GEMM) -> n_lstm x fused LSTM layer (b200_lstm_fused_tile_fwd) -> LinearCRFEncoder
 * GEMM (+Clamp), enqueued on `stream` (9 launches for the hac shape).  Replaces the module-tree walk of
 * `Serial.forward` over the encoder of a bonito.crf model (bonito/nn.py:82-89, bonito/crf/model.py:150-162) -- the span
 * `Model.use_koi` swaps for koi.lstm.update_graph plus the layers around it.  Tile-layout recurrent kernel only
 * (b200_lstm_tile_chunks(hidden) > 0).  The plan holds DEVICE pointers to packed weights (layouts as documented for the
 * fine-grained entry points above: conv weights in torch layout, w3 [H][k3*c2] with k = tap*c2 + cin, wih / bias in gx column
 * order, whh in W_hh row order) and to caller-owned work buffers:
 *   stem  (n*tp*s3*c2 + k3*c2) halves, the last k3*c2 zeroed       ya, yb  tiles*t*64*H halves, zero-filled once
 *   gx    unused (may be NULL)                                      hx      b200_lstm_rec_tile_workspace_bytes(n) bytes
 * with tiles = ceil(n / 64), t = frames, tp = padded frames per chunk (the stem buffer holds tp*s3 samples per chunk).
 * x [n][l] fp16 -> scores [n][t][n_scores] fp16 (no blank column).
 */
#define B200_MAX_LSTM_LAYERS 8
typedef struct b200_lstm_crf_plan {
    int n, l, t, tp;
    int c1, k1, act1, c2, k2, act2;          /* conv stem */
    int hidden, k3, s3, pad3, act3;          /* strided convolution into the LSTM width */
    int n_lstm, n_scores, act_l;
    float lo, hi;                            /* clamp bounds (act_l = B200_ACT_CLAMP) */
    int reverse[B200_MAX_LSTM_LAYERS];
    const void *w1, *b1, *w2, *b2, *w3, *b3, *wl, *bl;
    const void* wih[B200_MAX_LSTM_LAYERS];
    const void* bias[B200_MAX_LSTM_LAYERS];
    const void* whh[B200_MAX_LSTM_LAYERS];
    void *stem, *ya, *yb, *gx, *hx;
} b200_lstm_crf_plan;
int b200_lstm_crf_fwd(const b200_lstm_crf_plan* plan, const void* x, void* scores, void* stream);

/*
 * Beam-search decode with the argument meaning of koi.decode.beam_search (bonito/crf/basecall.py:36-40): beam_width entries
 * (1..32), candidates more than beam_cut (natural-log units) below the best are dropped.  koi itself is a closed binary with
 * no pinned outputs, so this is this library's own backward-guided prefix beam search (oracle: crf_oracle.beam_search_native);
 * the exact posterior-Viterbi decoder b200_crf_decode stays the default.  Same scores / outputs / workspace as b200_crf_decode
 * (the forward-backward pass runs first and provides the look-ahead scores and the qualities).
 */
int b200_crf_beam_search(const void* scores, int n, int t, int state_len, float blank_score, int beam_width, float beam_cut,
                         float qscale, float qbias, void* workspace, void* moves, void* sequence, void* qstring, void* stream);

/*
 * ---- CTC-CRF sequence distribution (reference: CTC_CRF, bonito/crf/model.py:30-143, on koi.ctc's logZ_cu_sparse,
 *      fwd/bwd_scores_cu_sparse, logZ_cu and viterbi_alignments) ----
 * All tensors fp32 (lengths int32), contiguous, on the device; `semiring` is B200_SEMIRING_LOG (logsumexp) or
 * B200_SEMIRING_MAX.  Every output is written in full and is bitwise reproducible.
 *
 * The k-mer lattice: S = 4^state_len states (state_len 1..5), scores [t][n][5*S] 16-byte aligned, the edge from
 * idx[s][e] into s at column s*5 + e (idx[s][0] = s, idx[s][1+j] = j*S/4 + s/4); alpha_0 = beta_t = 0 for every state.
 *   b200_ctc_crf_sparse_fwd:  logz [n]; alpha [t+1][n][S] when not NULL; when `workspace` is not NULL (of
 *     b200_ctc_crf_sparse_workspace_bytes(n, t, state_len, semiring) bytes) it keeps what b200_ctc_crf_sparse_grad needs.
 *   b200_ctc_crf_sparse_bwd:  beta [t+1][n][S].
 *   b200_ctc_crf_sparse_grad: grad [t][n][5*S] = g[c] * dlogz[c]/dscores from the workspace of a forward with the same
 *     arguments.  Log: g * exp(alpha_t[idx[s][e]] + scores[t][c][s*5+e] + beta_{t+1}[s] - logz); Max: g on the edges of
 *     the best path (ties: the lowest in-edge at every frame, then the lowest final state), 0 elsewhere.
 *
 * The target lattice of ctc_loss: stay [t][n][l], move [t][n][l-1], lengths [n] (target_lengths + 1 - state_len), l <=
 * b200_ctc_crf_target_max_states();  alpha_0 = [0, -inf, ...], alpha_{u+1}[j] = alpha_u[j] * stay[u][j] (+)
 * alpha_u[j-1] * move[u][j-1] (semiring product and sum), logz = alpha_t[lengths-1].  A chunk with lengths < 1,
 * lengths > l or lengths - 1 > t is infeasible: logz = -inf and a gradient of exactly 0.
 *   b200_ctc_crf_target_fwd:  logz [n]; `workspace` (b200_ctc_crf_target_workspace_bytes bytes) as above, or NULL.
 *   b200_ctc_crf_target_grad: dstay [t][n][l], dmove [t][n][l-1] = g[c] * dlogz[c]/d(stay, move); Max: g on the edges
 *     of the best path, ties to the stay.
 */
#define B200_SEMIRING_LOG 0
#define B200_SEMIRING_MAX 1
size_t b200_ctc_crf_sparse_workspace_bytes(int n, int t, int state_len, int semiring);
int b200_ctc_crf_sparse_fwd(const void* scores, int t, int n, int state_len, int semiring, void* logz, void* alpha,
                            void* workspace, void* stream);
int b200_ctc_crf_sparse_bwd(const void* scores, int t, int n, int state_len, int semiring, void* beta, void* stream);
int b200_ctc_crf_sparse_grad(const void* scores, int t, int n, int state_len, int semiring, const void* g,
                             void* workspace, void* grad, void* stream);
int b200_ctc_crf_target_max_states(void);
size_t b200_ctc_crf_target_workspace_bytes(int n, int t, int l, int semiring);
int b200_ctc_crf_target_fwd(const void* stay, const void* move, const void* lengths, int t, int n, int l, int semiring,
                            void* logz, void* workspace, void* stream);
int b200_ctc_crf_target_grad(const void* stay, const void* move, const void* lengths, int t, int n, int l, int semiring,
                             const void* g, void* workspace, void* dstay, void* dmove, void* stream);

/*
 * ---- CTC prefix beam search (reference: fast_ctc_decode.beam_search behind bonito/ctc/model.py:39-46; that crate's output
 *      is pinned by nothing here, so the cut, merge, tie, move and quality rules are this library's, stated in
 *      bonito_b200/csrc/ctc_beam.cu) ----
 * logp: DEVICE fp16 [frames][5] log-probs (class 0 = blank, 1..4 = A C G T) of n_reads reads packed along the frame axis;
 * read r is frames [frame_off[r], frame_off[r] + frame_len[r]).  As for b200_sw_align, frame_off (int64) and frame_len
 * (int32) are HOST arrays, checked on the host (0 <= frame_len <= 2^26, else -2) and copied into the head of `workspace`
 * on `stream`.  beam_width in [1, 32]; a class whose probability is below `threshold` (in [0, 1], the reference uses 1e-3)
 * is skipped at that frame.
 * workspace: DEVICE memory of workspace_bytes >= b200_ctc_beam_workspace_bytes(n_reads, sum of frame_len, beam_width)
 * bytes (the per-read arrays plus 1 + beam_width * frame_len[r] prefix nodes of 8 bytes per read); a smaller one returns
 * -2 with the sizes in the message before anything is launched.
 * sequence / qstring / moves: DEVICE bytes indexed like the frames of logp; every frame of every read is written: the base
 * ('A' 'C' 'G' 'T'), its quality character and 1 on the frame where a base of the answer entered the beam, 0 elsewhere
 * (the byte layout of b200_crf_decode).  Frames outside the reads are not touched.  Bitwise reproducible.
 */
size_t b200_ctc_beam_workspace_bytes(int n_reads, long long total_frames, int beam_width);
int b200_ctc_beam_search(const void* logp, const long long* frame_off, const int* frame_len, int n_reads, int beam_width,
                         float threshold, float qscale, float qbias, void* workspace, size_t workspace_bytes, void* sequence,
                         void* qstring, void* moves, void* stream);

/*
 * ---- read-to-reference mapping for `basecaller --reference` (the reference maps with minimap2 through mappy; the
 *      minimizer, anchor, chaining, extraction and alignment rules here are this library's, stated in
 *      bonito_b200/csrc/map.cu).  Every array is DEVICE memory; int64 unless stated. ----
 * b200_map_minimizers: seq = n_seqs sequences packed back to back, sequence s at [seq_off[s], seq_off[s + 1]); odd k in
 *   [3, 31], w in [1, 255].  kmer (scratch) and mm are [n_bases]; mm[p] = hash << 1 | strand of the minimizer at p, else -1.
 * b200_map_anchors: index = uniq [n_unique] (sorted hashes), start [n_unique + 1], val [start[n_unique]] (position << 1 |
 *   strand); a hash with more than max_occ entries is skipped.  count != NULL: count (int32 [n_bases]) = anchors per
 *   position, nothing else written.  count == NULL: aoff [n_bases] (exclusive prefix of count) places each position's
 *   anchors: akey = read << 33 | strand << 32 | reference position, aq (int32) = query position on that strand.
 * b200_map_chain: anchors sorted by akey; read r owns [read_aoff[r], read_aoff[r + 1]); contigs are [ctg_off[c],
 *   ctg_off[c + 1]) of the global reference coordinate.  f, pred: int32 [anchors].
 * b200_map_extract: order = the anchors sorted by (read, decreasing f, index); taken = uint8 [anchors], zeroed;
 *   chain = [anchors][2] receives the primary chain's (q, r) of read r at its anchor offset; out = [n_reads][9]: anchors in
 *   the primary chain, f1, f2, strand, band half-width (<= max_band), q / r of its first and of its last anchor.
 * b200_map_align: meta = [n_pairs][9]: query offset, m, target offset, n, chain pair offset, chain length, band half-width
 *   (<= max_band <= 4096), trace byte offset, ops slot offset (m + n bytes).  cen = int32 indexed like query; trace =
 *   b200_map_align_trace_bytes(m, band) bytes per pair.  out int32 [n_pairs][6] = score, q_st, q_en, t_st, t_en, n_ops; the
 *   ops ('=', 'X', 'I', 'D', forward order) are the last n_ops bytes of the pair's slot.
 */
int b200_map_minimizers(const void* seq, long long n_bases, const long long* seq_off, int n_seqs, int k, int w, void* kmer,
                        void* mm, void* stream);
int b200_map_anchors(const void* mm, long long n_bases, const long long* seq_off, int n_seqs, int k, const void* uniq,
                     long long n_unique, const void* start, const void* val, int max_occ, void* count, const void* aoff,
                     void* akey, void* aq, void* stream);
int b200_map_chain(const void* akey, const void* aq, const long long* read_aoff, int n_reads, const long long* ctg_off, int n_ctg,
                   int k, void* f, void* pred, void* stream);
int b200_map_extract(const void* akey, const void* aq, const void* f, const void* pred, const void* order,
                     const long long* read_aoff, const long long* seq_off, int n_reads, int k, int max_band, void* taken,
                     void* chain, void* out, void* stream);
size_t b200_map_align_trace_bytes(int query_len, int band);
int b200_map_align(const void* query, const void* target, const void* chain, const void* meta, int n_pairs, int max_band,
                   void* cen, void* trace, void* ops, void* out, void* stream);

/*
 * ---- BGZF compression for BAM output (SAM specification section 4.1; the DEFLATE parse and codes are this library's,
 *      stated in bonito_b200/csrc/bgzf.cu) ----
 * in: DEVICE bytes [in_bytes], cut into n = ceil(in_bytes / B200_BGZF_MEMBER_INPUT) members in order, each of
 * B200_BGZF_MEMBER_INPUT bytes but the last (in_bytes == 0: no members).  Every member is one gzip member with the BC
 * extra subfield (BSIZE = member size - 1), one final DEFLATE block (dynamic Huffman codes, or stored when that is not
 * larger), CRC32 and ISIZE; the members are written back to back into out (DEVICE, capacity n * 65536 bytes) and
 * out_offsets (DEVICE int64 [n + 1]) receives their start offsets and, last, the total length.  The 28-byte EOF marker is
 * the caller's.  workspace: DEVICE memory of b200_bgzf_workspace_bytes(in_bytes) bytes.  Byte-identical from run to run.
 */
#define B200_BGZF_MEMBER_INPUT 65280 /* htslib's BGZF_BLOCK_SIZE (0xff00): a stored member still fits in 64 KiB */
size_t b200_bgzf_workspace_bytes(int64_t in_bytes);
int b200_bgzf_compress(const uint8_t* in, int64_t in_bytes, uint8_t* out, int64_t* out_offsets, void* workspace,
                       size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BONITO_B200_H */
