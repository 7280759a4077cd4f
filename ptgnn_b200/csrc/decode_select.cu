// Per-graph token selection of graph2seq's greedy decoding (the reference's GruCopyingDecoderModel.greedy_decode,
// grucopydecoder.py:406-455), one CTA per graph, for one decoder step:
//   1. Z = logsumexp(x ∪ {lse_copy[g]}) with x = logits[g, :V]: a block max, then a block sum of expf(x - max), both in a fixed
//      tree order (strided per-thread partials, xor butterflies, warps in order).  lp_v = fl(x_v - Z), c_i = fl(s_i - Z).
//   2. T = the K = min(100, V) largest lp, the lower id first among equal values: a radix select over order-preserving uint32 keys of
//      lp, four passes of 8-bit digits with shared-memory histograms, gives the K-th key (the threshold) and how many ids equal to it
//      are admitted.  When the threshold's ties are split, one more pass finds the highest admitted id.  Membership is then a
//      comparison.  The first pass also finds the top-1 (largest lp, lowest id).
//   3. One pass over the graph's copy groups (rows sharing a key, in first-occurrence order, rows in row order): a group scores
//      lp_key ⊕ c_i1 ⊕ c_i2 ... when its key is in T, else c_i1 ⊕ c_i2 ..., with ⊕ numpy's float32 logaddexp applied in row order.
//   4. A block argmax over the top-1 and the groups: the higher score wins; a tie goes to the earlier entry of the reference's
//      dictionary: members of T first (larger lp, then lower id), then the groups outside T in first-occurrence order.  A member of T
//      without a group scores its lp <= the top-1's, so it never needs a candidate of its own.
//   5. Thread 0 updates the graph's state: a done graph feeds END and keeps its log-probability and tokens; otherwise the score is
//      added to the fp32 log-probability, END marks the graph done, any other key is appended, and the next input id is the key when
//      it is below V, else UNK.
// No float atomics, no host synchronisation: results are bit-identical from run to run.  Error bounds: DESIGN.md §3.18.  Steps 1-3
// are the helpers of decode_select.cuh, shared with beam search (beam_select.cu).
#include "common.cuh"
#include "decode_select.cuh"

namespace ptgnn {
namespace decode_select {

__global__ void __launch_bounds__(THREADS, 1) decode_select_kernel(
    const float *__restrict__ logits, int V, const float *__restrict__ copy_scores, const float *__restrict__ lse_copy,
    const int32_t *__restrict__ group_ptr, const int32_t *__restrict__ group_key, const int32_t *__restrict__ member_ptr,
    const int32_t *__restrict__ member_rows, int end_id, int unk_id, int step, int max_len, int32_t *__restrict__ done,
    int32_t *__restrict__ length, float *__restrict__ logprob, int32_t *__restrict__ tokens, int64_t *__restrict__ next_ids,
    float *__restrict__ stats) {
    __shared__ Smem sm;
    const int g = blockIdx.x, tid = threadIdx.x;
    const bool was_done = step > 0 && done[g] != 0;
    if (was_done) {                     // uniform over the block: nothing to select
        if (tid == 0) {
            next_ids[g] = end_id;
            stats[2 * g] = stats[2 * g + 1] = __int_as_float(0x7fc00000);
        }
        return;
    }
    const float *x = logits + (long long)g * V;

    // 1. the normaliser
    const float Z = row_normaliser(x, V, lse_copy[g], sm);

    // 2. radix select of the K-th largest key of lp, and the top-1
    uint32_t best_key;
    int best_id;
    const uint32_t thr = radix_select_top(x, V, Z, sm, best_key, best_id);
    Cand top = NONE;                    // a thread without ids (V < THREADS) holds no candidate
    if (best_id < V) {
        top.score = key_value(best_key);
        top.cls = 0;
        top.a = ~best_key;
        top.b = (uint32_t)best_id;
        top.key = best_id;
    }
    top = block_best(top, sm);          // also orders the write of sm.id_cut before its reads
    const uint32_t id_cut = sm.id_cut;

    // 3. the copy groups, 4. the argmax
    Cand c = tid == 0 ? top : NONE;
    const int g0 = group_ptr[g], g1 = group_ptr[g + 1];
    for (int j = g0 + tid; j < g1; j += THREADS) {
        const Cand d = group_entry(x, V, Z, thr, id_cut, j, g0, group_key[j], member_ptr, member_rows, copy_scores, 1);
        if (better(d, c)) c = d;
    }
    c = block_best(c, sm);

    // 5. the state update
    if (tid == 0) {
        const int len = step > 0 ? length[g] : 0;
        const float lp = (step > 0 ? logprob[g] : 0.0f) + c.score;
        logprob[g] = lp;
        if (c.key == end_id) {
            done[g] = 1;
            length[g] = len;
        } else {
            done[g] = 0;
            if (len < max_len) tokens[(long long)g * max_len + len] = c.key;
            length[g] = min(len + 1, max_len);
        }
        next_ids[g] = c.key < V ? c.key : unk_id;
        stats[2 * g] = Z;
        stats[2 * g + 1] = c.score;
    }
}

}  // namespace decode_select
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_decode_select_supported(int32_t vocab) { return decode_select::supported(vocab) ? 1 : 0; }

extern "C" size_t ptgnn_b200_decode_select_workspace_bytes(int64_t num_graphs, int32_t vocab) {
    if (num_graphs < 0 || !decode_select::supported(vocab)) return 0;
    return ws_slice((size_t)num_graphs * 2, 4);
}

extern "C" int ptgnn_b200_decode_select(const float *logits, int64_t num_graphs, int32_t vocab, const float *copy_scores, int64_t num_rows,
                                        const float *lse_copy, const int32_t *group_ptr, const int32_t *group_key, const int32_t *member_ptr,
                                        const int32_t *member_rows, int32_t end_id, int32_t unk_id, int32_t step, int32_t max_len,
                                        int32_t *done, int32_t *length, float *logprob, int32_t *tokens, int64_t *next_ids, void *workspace,
                                        size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!decode_select::supported(vocab)) {
        set_error("decode_select: vocabulary size %d not supported (1 to %d)", vocab, decode_select::MAX_VOCAB);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_graphs >= 0 && num_graphs < INT32_MAX && num_rows >= 0 && num_rows < INT32_MAX, "decode_select: sizes out of range");
    PTGNN_CHECK_ARG(step >= 0 && step < max_len, "decode_select: step %d outside [0, max_len = %d)", step, max_len);
    PTGNN_CHECK_ARG(end_id >= 0 && end_id < vocab && unk_id >= 0 && unk_id < vocab, "decode_select: end_id / unk_id outside the vocabulary");
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(logits && lse_copy && group_ptr && done && length && logprob && tokens && next_ids && (num_rows == 0 || copy_scores),
                    "decode_select: null pointer");
    PTGNN_CHECK_WORKSPACE("decode_select", workspace, workspace_bytes, ptgnn_b200_decode_select_workspace_bytes(num_graphs, vocab));
    return launch(PTGNN_KERNEL_REDUCE, st, decode_select::decode_select_kernel, (unsigned)num_graphs, decode_select::THREADS, 0, logits,
                  (int)vocab, copy_scores, lse_copy, group_ptr, group_key, member_ptr, member_rows, (int)end_id, (int)unk_id, (int)step,
                  (int)max_len, done, length, logprob, tokens, next_ids, static_cast<float *>(workspace));
}
