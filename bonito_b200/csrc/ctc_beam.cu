// CTC prefix beam search for the QuartzNet CTC models (`beamsize > 1` of bonito_b200.ctc; the reference calls the CPU
// crate fast_ctc_decode, bonito/ctc/model.py:39-46, whose output nothing here pins, so the rules below are this library's).
//
// Definition (the CPU oracle, tests/_oracle_ctc_beam.py, states the same rules with float64 sums over prefix tuples):
//   input   one read = T frames of 5 fp16 log-probs, class 0 = blank; p[c] = exp(logp[t][c]) rounded to fp32.
//   beam    entries (node, p_label, p_blank), ranked by p_label + p_blank; a node is a prefix (parent, label,
//           frame_created).  It starts as the empty prefix with p_label = 0, p_blank = 1.
//   cut     a class with p[c] < threshold is skipped at that frame, the blank included; a frame whose five classes are all
//           skipped leaves the beam as it is.
//   frame   every entry proposes, for every class c that is not skipped:
//             c = blank                 its own node,  p_blank' += (p_label + p_blank) p[0]
//             c = its last label        its own node,  p_label' += p_label p[c];  its child c,  p_label' += p_blank p[c]
//             any other label c         its child c,   p_label' += (p_label + p_blank) p[c]
//           Proposals for the same prefix are summed.  A child that is already an entry of the beam is that entry: the
//           proposal joins the entry's own ones (entry B is the child c of entry A when parent(B) = node(A) and
//           label(B) = c).  A prefix is a candidate when its summed total p_label' + p_blank' is > 0; a frame without
//           a candidate leaves the beam as it is.
//   select  the beam_width candidates with the largest total; ties go to the candidate whose proposing entry had the
//           lower rank in the previous beam (for a kept node: its own rank), then to the kept node before the children,
//           then to the lower class.  The new beam is ranked in that order and divided by its top total, so the values
//           stay in range however long the read is.
//   nodes   only surviving children are written to the arena, at most beam_width per frame, with frame_created = the
//           frame at which they entered the beam.  A prefix that left the beam and is proposed again is a new node:
//           descendants of the old one that are still in the beam are not its children.
//   answer  the prefix of the top entry after the last frame: walking `parent` gives the bases and their frames, which
//           increase strictly, so `moves` is 1 exactly on those frames and `sequence` holds the base there.
//   quality the span of base i is [frame_i, frame_{i+1}) (the last one ends with the read); q_i = phred of the mean of p[l_i]
//           over the frames of the span whose argmax is l_i (equal log-probs: the highest index wins, as in b200_ctc_head_fwd;
//           no such frame: the emission frame alone), the mean in float64, phred(p) = clip(rint(-10 log10(max(1 - p, 1e-4))
//           * qscale + qbias) + 33, 33, 126).  With the bases and frames of the greedy decode this is the greedy quality.
//
// Shape: the search is sequential in T, so one warp owns one read (reads grid-strided over one-warp CTAs) and lanes are beam
// entries, lane = rank.  Frames arrive in blocks of 32: lane l loads and exponentiates frame t0 + l into shared memory while
// the next block's 5 halves are already in flight.  Per frame every lane finds its parent's lane and the labels of its
// children in the beam with shuffles, forms its <= 5 candidates (kept node, children 1..4) as monotone uint keys
// (float bits + 1, 0 = none), and the warp extracts the best beam_width times: redux.sync max, ballot, lowest lane, lowest
// slot -- which is the tie rule.  The winner writes the new entry of that rank to shared memory; afterwards lane r takes
// entry r and new nodes get consecutive arena slots in rank order (ballot + popc).  No atomics, no dependence on the other
// reads of the launch: the result is bitwise reproducible.  Lane 0 walks the answer back and writes the label index into
// `qstring`; a second, frame-parallel kernel turns it into the quality.
#include <vector>

#include "common.cuh"

namespace {

constexpr int CB_NCLS = 5;
constexpr int CB_MAX_WIDTH = 32;
constexpr int CB_MAX_FRAMES = 1 << 26;     // per read: frame << 3 | label and 1 + 32 T node ids stay inside int32
constexpr int CB_QUAL_THREADS = 256;
constexpr unsigned FULL = 0xffffffffu;

struct BeamMeta {                          // the per-read arrays, in the head of the workspace
    const long long* off;                  // first frame of read r in logp / the outputs
    const long long* node_off;             // first arena node of read r
    const int* len;                        // frames of read r
};

size_t meta_bytes(int n_reads) { return (((size_t)n_reads * 20) + 255) & ~(size_t)255; }

__device__ __forceinline__ float prob_of(__half lp) { return (float)exp((double)__half2float(lp)); }

__global__ void __launch_bounds__(32)
ctc_beam_kernel(const __half* __restrict__ logp, BeamMeta meta, int n_reads, int width, float threshold,
                int2* __restrict__ arena, uint8_t* __restrict__ seq, uint8_t* __restrict__ qual, uint8_t* __restrict__ moves) {
    __shared__ float s_p[32][CB_NCLS];                       // p[c] of the 32 frames of the current block
    __shared__ int s_node[32], s_par[32], s_last[32];        // the new beam, by rank
    __shared__ float s_pl[32], s_pb[32];
    const int lane = threadIdx.x;
    for (int r = blockIdx.x; r < n_reads; r += gridDim.x) {
        const int T = meta.len[r];
        if (T == 0) continue;
        const long long base = meta.off[r];
        int2* nodes = arena + meta.node_off[r];
        for (int t = lane; t < T; t += 32) seq[base + t] = 0, qual[base + t] = 0, moves[base + t] = 0;
        if (lane == 0) nodes[0] = make_int2(-1, 0);
        int count = 1, n = 1;                                // arena nodes in use, beam entries
        int node = lane == 0 ? 0 : -2, par = lane == 0 ? -1 : -3, last = 0;
        float pl = 0.f, pb = lane == 0 ? 1.f : 0.f;
        __half h[CB_NCLS];
        if (lane < T) {
#pragma unroll
            for (int c = 0; c < CB_NCLS; ++c) h[c] = logp[(base + lane) * CB_NCLS + c];
        }
        for (int t0 = 0; t0 < T; t0 += 32) {
            __syncwarp();
#pragma unroll
            for (int c = 0; c < CB_NCLS; ++c) s_p[lane][c] = t0 + lane < T ? prob_of(h[c]) : 0.f;
            __syncwarp();
            if (t0 + 32 + lane < T) {
#pragma unroll
                for (int c = 0; c < CB_NCLS; ++c) h[c] = logp[(base + t0 + 32 + lane) * CB_NCLS + c];
            }
            const int nb = min(32, T - t0);
            for (int k = 0; k < nb; ++k) {
                float p[CB_NCLS];
                unsigned alive = 0;
#pragma unroll
                for (int c = 0; c < CB_NCLS; ++c) {
                    p[c] = s_p[k][c];
                    if (!(p[c] < threshold)) alive |= 1u << c;
                }
                if (alive == 0) continue;
                // the lane holding this entry's parent, and the labels of this entry's children that are in the beam
                int plane = -1;
                unsigned child = 0;
                for (int j = 0; j < n; ++j) {
                    const int nj = __shfl_sync(FULL, node, j), pj = __shfl_sync(FULL, par, j), lj = __shfl_sync(FULL, last, j);
                    if (par == nj) plane = j;
                    if (pj == node) child |= 1u << lj;
                }
                const bool active = lane < n;
                const float tot = pl + pb;
                const bool last_alive = last != 0 && ((alive >> last) & 1u);
                const float p_last = s_p[k][last];
                // the kept node: blank, its own last label, and its last label proposed by its parent
                float kpl = 0.f, kpb = 0.f;
                bool keep = false;
                if (active && (alive & 1u)) kpb = tot * p[0], keep = true;
                if (active && last_alive) kpl = pl * p_last, keep = true;
                const int src = plane < 0 ? 0 : plane;
                const float ppl = __shfl_sync(FULL, pl, src), ppb = __shfl_sync(FULL, pb, src);
                const int plast = __shfl_sync(FULL, last, src);
                if (active && plane >= 0 && last_alive) kpl += (plast == last ? ppb : ppl + ppb) * p_last, keep = true;
                unsigned key[CB_NCLS];
                key[0] = keep && kpl + kpb > 0.f ? __float_as_uint(kpl + kpb) + 1u : 0u;
#pragma unroll
                for (int c = 1; c < CB_NCLS; ++c) {
                    const bool is = active && ((alive >> c) & 1u) && !((child >> c) & 1u);
                    const float v = (c == last ? pb : tot) * p[c];
                    key[c] = is && v > 0.f ? __float_as_uint(v) + 1u : 0u;
                }
                int nn = 0;
                float top = 0.f;
                for (int rank = 0; rank < width; ++rank) {
                    unsigned best = key[0];
                    int slot = 0;
#pragma unroll
                    for (int c = 1; c < CB_NCLS; ++c)
                        if (key[c] > best) best = key[c], slot = c;
                    const unsigned m = __reduce_max_sync(FULL, best);
                    if (m == 0) break;
                    const int winner = __ffs(__ballot_sync(FULL, best == m)) - 1;
                    if (lane == winner) {
                        if (slot == 0) {
                            s_node[rank] = node, s_par[rank] = par, s_last[rank] = last, s_pl[rank] = kpl, s_pb[rank] = kpb;
                        } else {
                            s_node[rank] = -1, s_par[rank] = node, s_last[rank] = slot;
                            s_pl[rank] = __uint_as_float(best - 1u), s_pb[rank] = 0.f;
                        }
#pragma unroll
                        for (int c = 0; c < CB_NCLS; ++c)
                            if (c == slot) key[c] = 0;
                    }
                    if (rank == 0) top = __uint_as_float(m - 1u);
                    ++nn;
                }
                __syncwarp();
                if (nn == 0) continue;
                n = nn;
                const float inv = 1.0f / top;
                if (lane < n) {
                    node = s_node[lane], par = s_par[lane], last = s_last[lane];
                    pl = s_pl[lane] * inv, pb = s_pb[lane] * inv;
                } else {
                    node = -2, par = -3, last = 0, pl = 0.f, pb = 0.f;
                }
                const unsigned fresh = __ballot_sync(FULL, node == -1);
                if (node == -1) {
                    node = count + __popc(fresh & ((1u << lane) - 1u));
                    nodes[node] = make_int2(par, ((t0 + k) << 3) | last);
                }
                count += __popc(fresh);
                __syncwarp();
            }
        }
        __syncwarp();
        if (lane == 0) {
            for (int id = node; id > 0;) {
                const int2 nd = nodes[id];
                const long long at = base + (nd.y >> 3);
                const int l = nd.y & 7;
                seq[at] = (uint8_t)"NACGT"[l], qual[at] = (uint8_t)l, moves[at] = 1;
                id = nd.x;
            }
        }
        __syncwarp();
    }
}

// One thread per emitting frame scans its span; `qual` holds the label index on entry and the quality on exit.
__global__ void __launch_bounds__(CB_QUAL_THREADS)
ctc_beam_qual_kernel(const __half* __restrict__ logp, BeamMeta meta, int n_reads, float qscale, float qbias,
                     uint8_t* __restrict__ qual, const uint8_t* __restrict__ moves) {
    for (int r = blockIdx.y; r < n_reads; r += gridDim.y) {
        const int T = meta.len[r];
        const long long base = meta.off[r];
        for (int t = blockIdx.x * CB_QUAL_THREADS + threadIdx.x; t < T; t += gridDim.x * CB_QUAL_THREADS) {
            if (!moves[base + t]) continue;
            const int l = qual[base + t];
            double sum = 0.0;
            int cnt = 0;
            for (int u = t; u < T && (u == t || !moves[base + u]); ++u) {
                const __half* row = logp + (base + u) * CB_NCLS;
                int best = 0;
                float top = -INFINITY;
#pragma unroll
                for (int c = 0; c < CB_NCLS; ++c) {
                    const float v = __half2float(row[c]);
                    if (v >= top) top = v, best = c;
                }
                if (best == l) sum += (double)prob_of(row[l]), ++cnt;
            }
            if (cnt == 0) sum = (double)prob_of(logp[(base + t) * CB_NCLS + l]), cnt = 1;
            const double err = fmax(1.0 - sum / cnt, 1e-4);
            const double q = rint(-10.0 * log10(err) * (double)qscale + (double)qbias) + 33.0;
            qual[base + t] = (uint8_t)fmin(fmax(q, 33.0), 126.0);
        }
    }
}

}  // namespace

size_t ctc_beam_workspace_bytes(int n_reads, long long total_frames, int beam_width) {
    if (n_reads <= 0 || total_frames < 0 || beam_width < 1 || beam_width > CB_MAX_WIDTH) return 0;
    return meta_bytes(n_reads) + ((size_t)n_reads + (size_t)beam_width * (size_t)total_frames) * sizeof(int2);
}

int launch_ctc_beam_search(const __half* logp, const long long* frame_off, const int* frame_len, int n_reads, int beam_width,
                           float threshold, float qscale, float qbias, void* workspace, size_t workspace_bytes,
                           uint8_t* sequence, uint8_t* qstring, uint8_t* moves, cudaStream_t stream) {
    B200_REQUIRE(n_reads >= 0, "ctc_beam_search: bad read count %d", n_reads);
    B200_REQUIRE(beam_width >= 1 && beam_width <= CB_MAX_WIDTH, "ctc_beam_search: beam_width %d is outside [1, %d]",
                 beam_width, CB_MAX_WIDTH);
    B200_REQUIRE(threshold >= 0.f && threshold <= 1.f, "ctc_beam_search: threshold %g is outside [0, 1]", (double)threshold);
    if (n_reads == 0) return 0;
    B200_REQUIRE(frame_off && frame_len, "ctc_beam_search: null pointer argument");
    long long total = 0;
    int longest = 0;
    std::vector<long long> node_off((size_t)n_reads);
    for (int r = 0; r < n_reads; ++r) {
        B200_REQUIRE(frame_len[r] >= 0 && frame_len[r] <= CB_MAX_FRAMES,
                     "ctc_beam_search: read %d has %d frames; a read must have [0, %d]", r, frame_len[r], CB_MAX_FRAMES);
        B200_REQUIRE(frame_off[r] >= 0, "ctc_beam_search: read %d has a negative offset", r);
        node_off[r] = (long long)r + (long long)beam_width * total;
        total += frame_len[r];
        longest = frame_len[r] > longest ? frame_len[r] : longest;
    }
    if (total == 0) return 0;
    const size_t need = ctc_beam_workspace_bytes(n_reads, total, beam_width);
    B200_REQUIRE(workspace_bytes >= need,
                 "ctc_beam_search: the workspace has %zu bytes, %zu needed for %d reads of %lld frames at width %d "
                 "(1 + width * frames nodes per read)", workspace_bytes, need, n_reads, total, beam_width);
    B200_REQUIRE(logp && workspace && sequence && qstring && moves, "ctc_beam_search: null pointer argument");
    // the per-read arrays go into the head of the workspace: [off | node_off] int64, [len] int32
    char* head = static_cast<char*>(workspace);
    long long* off = reinterpret_cast<long long*>(head);
    long long* noff = off + n_reads;
    int* len = reinterpret_cast<int*>(noff + n_reads);
    B200_CHECK_CUDA(cudaMemcpyAsync(off, frame_off, sizeof(long long) * n_reads, cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(noff, node_off.data(), sizeof(long long) * n_reads, cudaMemcpyHostToDevice, stream));
    B200_CHECK_CUDA(cudaMemcpyAsync(len, frame_len, sizeof(int) * n_reads, cudaMemcpyHostToDevice, stream));
    const BeamMeta meta{off, noff, len};
    int2* arena = reinterpret_cast<int2*>(head + meta_bytes(n_reads));
    ctc_beam_kernel<<<(unsigned)n_reads, 32, 0, stream>>>(logp, meta, n_reads, beam_width, threshold, arena, sequence, qstring,
                                                          moves);
    B200_CHECK_CUDA(cudaGetLastError());
    const dim3 grid((unsigned)std::min(64, (longest + CB_QUAL_THREADS - 1) / CB_QUAL_THREADS), (unsigned)std::min(n_reads, 65535));
    ctc_beam_qual_kernel<<<grid, CB_QUAL_THREADS, 0, stream>>>(logp, meta, n_reads, qscale, qbias, qstring, moves);
    B200_CHECK_CUDA(cudaGetLastError());
    return 0;
}
