// Beam search of graph2seq (DESIGN.md §3.19): the selection of one decoder step over the K hypotheses ("slots") of every graph, in two
// kernels, with the decoding state on the device.
//
// beam_candidates_kernel, one 1024-thread CTA per (graph g, slot k):
//   * an empty slot has no candidate; a done slot has one, itself (key -1: nothing appended), with its total unchanged;
//   * a live slot builds the reference's dictionary for its row of logits exactly as greedy decoding does (decode_select.cuh): Z, T,
//     the copy groups with their float32 logaddexp scores.  Its K best entries in greedy's order (score descending, then members of T by
//     lp descending and id ascending, then groups outside T in first-occurrence order) are taken from the K best members of T that have
//     no group, by (lp, id), and every group: a member of T beyond those K is preceded by all of them, so it never reaches the K best.
//     The members of T without a group are first compacted into shared memory (at most 100); then K rounds of a block argmax each take
//     the best entry strictly after the previous round's winner in that total order, so no exclusion list is needed.  Each entry is
//     written with its score and its total fl(cum + score), in rank order.
// beam_merge_kernel, one 64-thread CTA per graph: the <= K^2 entries are ranked by (total descending, slot ascending, rank within the
//   slot ascending) -- each entry counts the entries before it, an exact integer rank -- and the K best become the new slots in rank
//   order.  It writes the step's backpointer and key tables, the totals, lengths, done and empty flags, the next input ids (the key when
//   below V, UNK for a copy outside the vocabulary, END for a done slot) and the gather index g·K + parent of the hidden-state reorder.
//   Slots beyond the number of candidates become empty.
// At step 0 the state is read as: slot 0 live with total 0 and length 0, the other slots empty.  No float atomics, no host
// synchronisation: results are bit-identical from run to run.
#include "common.cuh"
#include "decode_select.cuh"

namespace ptgnn {
namespace beam_select {

using namespace decode_select;

constexpr int MAX_BEAM = 8;
constexpr int MERGE_THREADS = MAX_BEAM * MAX_BEAM;

enum { LIVE = 0, DONE = 1, EMPTY = 2 };

// The state buffer (int32 words) of G graphs, K slots and max_len steps, in this order: backpointers [T][G][K], keys [T][G][K],
// totals [G][K] (fp32 bits), lengths [G][K], done flags [G][K], empty flags [G][K].
struct StateView {
    int32_t *bp, *key, *length, *done, *empty;
    float *total;
    __host__ __device__ StateView(int32_t *s, long long G, int K, int T) {
        const long long gk = G * K;
        bp = s;
        key = s + (long long)T * gk;
        total = reinterpret_cast<float *>(s + 2LL * T * gk);
        length = s + (2LL * T + 1) * gk;
        done = s + (2LL * T + 2) * gk;
        empty = s + (2LL * T + 3) * gk;
    }
};

// The workspace of G graphs and K slots: Z [G][K] fp32, counts [G][K] int32, then the entries [G][K][K]: keys int32, scores fp32,
// totals fp32.
struct Workspace {
    float *Z;
    int32_t *count;
    int32_t *key;
    float *score, *total;
};

inline size_t workspace_bytes(long long G, int K) {
    const size_t gk = (size_t)G * K, e = gk * K;
    return ws_slice(gk, 4) * 2 + ws_slice(e, 4) * 3;
}

inline Workspace carve(void *ws, long long G, int K) {
    const size_t gk = (size_t)G * K, e = gk * K;
    char *p = static_cast<char *>(ws);
    Workspace w;
    w.Z = reinterpret_cast<float *>(p);
    p += ws_slice(gk, 4);
    w.count = reinterpret_cast<int32_t *>(p);
    p += ws_slice(gk, 4);
    w.key = reinterpret_cast<int32_t *>(p);
    p += ws_slice(e, 4);
    w.score = reinterpret_cast<float *>(p);
    p += ws_slice(e, 4);
    w.total = reinterpret_cast<float *>(p);
    return w;
}

__device__ __forceinline__ int slot_status(const StateView &st, int step, long long gk, int k) {
    if (step == 0) return k == 0 ? LIVE : EMPTY;
    return st.empty[gk] ? EMPTY : st.done[gk] ? DONE : LIVE;
}

struct CandSmem {
    Smem base;
    uint32_t grouped[MAX_VOCAB / 32];    // bit v: the graph has a copy group with vocabulary key v
    uint32_t t_key[TOP_K];               // the members of T without a group: order_key of lp, and id
    int32_t t_id[TOP_K];
    int32_t t_count;
};

__global__ void __launch_bounds__(THREADS, 1) beam_candidates_kernel(
    const float *__restrict__ logits, int V, int K, const float *__restrict__ copy_scores, const float *__restrict__ lse_copy,
    const int32_t *__restrict__ group_ptr, const int32_t *__restrict__ group_key, const int32_t *__restrict__ member_ptr,
    const int32_t *__restrict__ member_rows, int step, int max_len, int32_t *__restrict__ state, int num_graphs, Workspace ws) {
    __shared__ CandSmem sm;
    const int g = blockIdx.x / K, k = blockIdx.x % K, tid = threadIdx.x;
    const long long gk = (long long)g * K + k;
    const StateView st(state, num_graphs, K, max_len);
    const int status = slot_status(st, step, gk, k);
    if (status != LIVE) {               // uniform over the block
        if (tid == 0) {
            ws.Z[gk] = __int_as_float(0x7fc00000);
            ws.count[gk] = status == DONE ? 1 : 0;
            if (status == DONE) {
                ws.key[gk * K] = -1;
                ws.score[gk * K] = 0.0f;
                ws.total[gk * K] = st.total[gk];
            }
        }
        return;
    }
    const float cum = step > 0 ? st.total[gk] : 0.0f;
    const float *x = logits + gk * V;

    const float Z = row_normaliser(x, V, lse_copy[gk], sm.base);
    uint32_t best_key;
    int best_id;
    const uint32_t thr = radix_select_top(x, V, Z, sm.base, best_key, best_id);

    // the vocabulary keys that have a group, and the members of T without one
    const int g0 = group_ptr[g], g1 = group_ptr[g + 1];
    for (int i = tid; i < (V + 31) / 32; i += THREADS) sm.grouped[i] = 0;
    if (tid == 0) sm.t_count = 0;
    __syncthreads();                    // also orders the write of sm.base.id_cut before its reads
    const uint32_t id_cut = sm.base.id_cut;
    for (int j = g0 + tid; j < g1; j += THREADS) {
        const int key = group_key[j];
        if (key < V) atomicOr(&sm.grouped[key >> 5], 1u << (key & 31));
    }
    __syncthreads();
    for (int v = tid; v < V; v += THREADS) {
        const uint32_t kv = order_key(x[v] - Z);
        if (in_top(kv, v, thr, id_cut) && !(sm.grouped[v >> 5] >> (v & 31) & 1u)) {
            const int at = atomicAdd(&sm.t_count, 1);      // the position is arbitrary: the rounds order by (lp, id)
            sm.t_key[at] = kv;
            sm.t_id[at] = v;
        }
    }
    __syncthreads();
    const int t_count = sm.t_count;

    // K rounds: each takes the best entry strictly after the previous winner
    Cand prev = NONE;
    int n = 0;
    for (int r = 0; r < K; ++r) {
        Cand c = NONE;
        for (int i = tid; i < t_count; i += THREADS) {
            Cand d;
            d.score = key_value(sm.t_key[i]);
            d.cls = 0;
            d.a = ~sm.t_key[i];
            d.b = (uint32_t)sm.t_id[i];
            d.key = sm.t_id[i];
            if ((r == 0 || better(prev, d)) && better(d, c)) c = d;
        }
        for (int j = g0 + tid; j < g1; j += THREADS) {
            const Cand d = group_entry(x, V, Z, thr, id_cut, j, g0, group_key[j], member_ptr, member_rows, copy_scores + k, K);
            if ((r == 0 || better(prev, d)) && better(d, c)) c = d;
        }
        c = block_best(c, sm.base);
        if (c.cls == 2) break;          // uniform: fewer than K entries
        if (tid == 0) {
            ws.key[gk * K + r] = c.key;
            ws.score[gk * K + r] = c.score;
            ws.total[gk * K + r] = cum + c.score;
        }
        prev = c;
        n = r + 1;
    }
    if (tid == 0) {
        ws.Z[gk] = Z;
        ws.count[gk] = n;
    }
}

__global__ void __launch_bounds__(MERGE_THREADS) beam_merge_kernel(int V, int K, int end_id, int unk_id, int step, int max_len,
                                                                   int32_t *__restrict__ state, int num_graphs, Workspace ws,
                                                                   int64_t *__restrict__ next_ids, int64_t *__restrict__ gather_idx) {
    __shared__ float tot[MERGE_THREADS];
    __shared__ int valid[MERGE_THREADS];
    __shared__ int old_len[MAX_BEAM];
    __shared__ int num_valid;
    const int g = blockIdx.x, t = threadIdx.x;
    const long long g0 = (long long)g * K;
    const StateView st(state, num_graphs, K, max_len);
    const int s = t / K, r = t % K;
    const bool mine = t < K * K && r < ws.count[g0 + s];
    tot[t] = mine ? ws.total[(g0 + s) * K + r] : 0.0f;
    valid[t] = mine;
    if (t < K) old_len[t] = step > 0 ? st.length[g0 + t] : 0;
    if (t == 0) num_valid = 0;
    __syncthreads();
    // the entry's rank: the entries before it by (total descending, index s·K + r ascending); its own index orders slot, then rank
    int rank = 0;
    if (mine) {
        for (int u = 0; u < K * K; ++u)
            if (valid[u] && (tot[u] > tot[t] || (tot[u] == tot[t] && u < t))) ++rank;
        atomicAdd(&num_valid, 1);
    }
    __syncthreads();                    // every read of the old lengths is done before the writes below
    const long long T_gk = (long long)step * num_graphs * K;
    if (mine && rank < K) {
        const long long j = g0 + rank;
        const int key = ws.key[(g0 + s) * K + r];
        st.bp[T_gk + j] = s;
        st.key[T_gk + j] = key;
        st.total[j] = tot[t];
        st.empty[j] = 0;
        if (key < 0 || key == end_id) {         // a done slot passing through, or END selected
            st.done[j] = 1;
            st.length[j] = old_len[s];
            next_ids[j] = end_id;
        } else {
            st.done[j] = 0;
            st.length[j] = min(old_len[s] + 1, max_len);
            next_ids[j] = key < V ? key : unk_id;
        }
        gather_idx[j] = g0 + s;
    }
    if (t < K && t >= min(num_valid, K)) {      // fewer than K entries: the remaining slots are empty
        const long long j = g0 + t;
        st.bp[T_gk + j] = -1;
        st.key[T_gk + j] = -1;
        st.total[j] = -INFINITY;
        st.length[j] = 0;
        st.done[j] = 0;
        st.empty[j] = 1;
        next_ids[j] = end_id;
        gather_idx[j] = j;
    }
}

bool supported(int64_t V, int64_t K) { return decode_select::supported(V) && K >= 1 && K <= MAX_BEAM; }

}  // namespace beam_select
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_beam_select_supported(int32_t vocab, int32_t beam_width) {
    return beam_select::supported(vocab, beam_width) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_beam_select_workspace_bytes(int64_t num_graphs, int32_t vocab, int32_t beam_width) {
    if (num_graphs < 0 || !beam_select::supported(vocab, beam_width)) return 0;
    return beam_select::workspace_bytes(num_graphs, beam_width);
}

extern "C" int ptgnn_b200_beam_select(const float *logits, int64_t num_graphs, int32_t vocab, int32_t beam_width, const float *copy_scores,
                                      int64_t num_rows, const float *lse_copy, const int32_t *group_ptr, const int32_t *group_key,
                                      const int32_t *member_ptr, const int32_t *member_rows, int32_t end_id, int32_t unk_id, int32_t step,
                                      int32_t max_len, int32_t *state, int64_t *next_ids, int64_t *gather_idx, void *workspace,
                                      size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!beam_select::supported(vocab, beam_width)) {
        set_error("beam_select: vocabulary size %d or beam width %d not supported (1 to %d, 1 to %d)", vocab, beam_width,
                  decode_select::MAX_VOCAB, beam_select::MAX_BEAM);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_graphs >= 0 && num_graphs * beam_width < INT32_MAX && num_rows >= 0 && num_rows * beam_width < INT32_MAX,
                    "beam_select: sizes out of range");
    PTGNN_CHECK_ARG(step >= 0 && step < max_len, "beam_select: step %d outside [0, max_len = %d)", step, max_len);
    PTGNN_CHECK_ARG(end_id >= 0 && end_id < vocab && unk_id >= 0 && unk_id < vocab, "beam_select: end_id / unk_id outside the vocabulary");
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(logits && lse_copy && group_ptr && state && next_ids && gather_idx && (num_rows == 0 || copy_scores),
                    "beam_select: null pointer");
    PTGNN_CHECK_WORKSPACE("beam_select", workspace, workspace_bytes, ptgnn_b200_beam_select_workspace_bytes(num_graphs, vocab, beam_width));
    const beam_select::Workspace ws = beam_select::carve(workspace, num_graphs, beam_width);
    int rc = launch(PTGNN_KERNEL_REDUCE, st, beam_select::beam_candidates_kernel, (unsigned)(num_graphs * beam_width),
                    decode_select::THREADS, 0, logits, (int)vocab, (int)beam_width, copy_scores, lse_copy, group_ptr, group_key, member_ptr,
                    member_rows, (int)step, (int)max_len, state, (int)num_graphs, ws);
    if (rc != PTGNN_OK) return rc;
    return launch(PTGNN_KERNEL_REDUCE, st, beam_select::beam_merge_kernel, (unsigned)num_graphs, beam_select::MERGE_THREADS, 0, (int)vocab,
                  (int)beam_width, (int)end_id, (int)unk_id, (int)step, (int)max_len, state, (int)num_graphs, ws, next_ids, gather_idx);
}
