"""graph2seq beam search on the GPU: beam width 1 against greedy decoding bit for bit, the selection kernels against the float64
restatement (beam_decode_reference.py) on constructed states, the whole decode at graph2seq's shape against the restatement driven
along the device's choices, re-scoring of every returned hypothesis, bit-identical reruns, no host synchronisation, a launch count per
step that depends on neither the number of steps nor the beam width, and the refusals.

Bounds are greedy decoding's (test_gpu_greedy_decode.py, DESIGN §3.18): a score within B_Z + (1 + 5 n) u (1 + |score|), doubled, plus
u |total| for the fp32 sum; a whole decode step within 2e-5 (1 + |score|).
"""
import math

import numpy as np
import pytest
import torch

import beam_decode_reference as BR
import greedy_decode_reference as GR
from test_gpu_greedy_decode import (STEP_BOUND, U, bounds, case, graph2seq_inputs, graph2seq_module, load, native_decode, quantised,
                                    seeded_module, vocab_of)

pytestmark = pytest.mark.gpu


# ---- the selection kernels ---------------------------------------------------------------------------------------------------------
def beam_case(V, G, K, gen):
    """Logits [G·K, V], copy scores [M, K] and lse [G, K] for K slots, with greedy's mix of copies (``case``)."""
    x, _, _, origin, values, vocab = case(V, G, gen)
    x = torch.cat([x] + [quantised(gen, (G, V)) for _ in range(K - 1)], 1).view(G * K, V)    # rows graph-major
    s = quantised(gen, (len(values), K), -6.0, 6.0)
    return x, s, lse_of(s, origin, G), origin, values, vocab


def lse_of(s, origin, G):
    s32 = s.float().double()
    lse = torch.full((G, s.shape[1]), -math.inf, dtype=torch.float64)
    for g in range(G):
        if (origin == g).any():
            lse[g] = torch.logsumexp(s32[origin == g], 0)
    return lse.float().double()


def new_state(G, K, V, max_len=4, start_id=1):
    from ptgnn_b200 import decoding

    return decoding.BeamState(G, K, max_len, V, start_id if V > 1 else 0, "cuda")


def set_state(state, total, done, empty, length=None):
    """Writes a constructed state (read by any step > 0)."""
    state.total.copy_(torch.as_tensor(total, dtype=torch.float32))
    state.done.copy_(torch.as_tensor(done, dtype=torch.int32))
    state.empty.copy_(torch.as_tensor(empty, dtype=torch.int32))
    state.length.copy_(torch.as_tensor(length if length is not None else np.zeros_like(np.asarray(done)), dtype=torch.int32))


def run_kernel(x, s, lse, origin, values, vocab, K, state, step, end_id=2, unk_id=0):
    from ptgnn_b200 import decoding

    G = lse.shape[0]
    groups = decoding.CopyGroups(values, origin.numpy(), G, vocab)
    before = state.buffer.clone()
    decoding.beam_select(x.float().cuda(), s.float().cuda().contiguous(), lse.float().cuda(), groups.to_device("cuda"), state, step,
                         end_id, unk_id)
    return before


def status_of(buffer_state, step, G, K):
    if step == 0:
        return [[BR.LIVE if k == 0 else BR.EMPTY for k in range(K)] for g in range(G)]
    empty, done = buffer_state
    return [[BR.EMPTY if empty[g][k] else BR.DONE if done[g][k] else BR.LIVE for k in range(K)] for g in range(G)]


def check_step(x, s, lse, origin, values, vocab, K, state, before, step, end_id=2, unk_id=0):
    """The kernels' selection, state and Z against the restatement.  Returns the restatement's merged lists."""
    G, V = lse.shape[0], x.shape[1]
    T = state.max_len
    gk = G * K
    old_total = before[2 * T * gk:(2 * T + 1) * gk].view(torch.float32).view(G, K).double().tolist()
    old_len = before[(2 * T + 1) * gk:(2 * T + 2) * gk].view(G, K).tolist()
    old_done = before[(2 * T + 2) * gk:(2 * T + 3) * gk].view(G, K).tolist()
    old_empty = before[(2 * T + 3) * gk:].view(G, K).tolist()
    status = status_of((old_empty, old_done), step, G, K)
    cum = old_total if step > 0 else [[0.0] * K for _ in range(G)]
    length = old_len if step > 0 else [[0] * K for _ in range(G)]
    keys = GR.row_keys(values, vocab)
    merged, Z = BR.step_from_logits(x.numpy(), s.numpy(), lse.numpy(), origin.numpy(), keys, status, cum, K)
    stats = state.stats().cpu().double()
    bp, kt = state.backpointers[step].cpu().tolist(), state.keys[step].cpu().tolist()
    tot, ln = state.total.cpu().double().tolist(), state.length.cpu().tolist()
    dn, em = state.done.cpu().tolist(), state.empty.cpu().tolist()
    nxt, gat = state.next_ids.cpu().view(G, K).tolist(), state.gather_idx.cpu().view(G, K).tolist()
    for g in range(G):
        for k in range(K):
            if status[g][k] == BR.LIVE:
                bz, _ = bounds(x[g * K + k:g * K + k + 1], torch.tensor([Z[g, k]]), torch.tensor([0.0]), torch.tensor([0.0]))
                assert abs(stats[g, k].item() - Z[g, k]) <= bz.item(), (g, k, stats[g, k].item(), Z[g, k])
            else:
                assert math.isnan(stats[g, k].item())
        m = merged[g]
        n_rows = int(np.bincount(origin.numpy(), minlength=G)[g])

        def tol(total, src):
            if math.isnan(Z[g, src]):   # a done slot's total is copied
                return 0.0
            _, bs = bounds(x[g * K + src:g * K + src + 1], torch.tensor([Z[g, src]]), torch.tensor([abs(total)]), torch.tensor([n_rows]))
            return bs.item() + U * abs(total)

        for j in range(K):
            if j >= len(m):
                assert em[g][j] == 1 and bp[g][j] == -1 and kt[g][j] == -1 and nxt[g][j] == end_id, (g, j)
                continue
            total, src, r, key = m[j]
            got = (bp[g][j], kt[g][j])
            if got != (src, key):
                # a near tie (never an exact one): the device's pick must be a candidate within the bounds of the restatement's
                alt = [e for e in m if (e[1], e[3]) == got]
                assert alt and 0 < abs(total - alt[0][0]) <= tol(total, src) + tol(alt[0][0], alt[0][1]), (g, j, got, (src, key), total)
                total, src, r, key = alt[0]
            assert abs(tot[g][j] - total) <= tol(total, src), (g, j, tot[g][j], total)
            assert em[g][j] == 0 and gat[g][j] == g * K + src
            if key == BR.DONE_KEY or key == end_id:
                assert dn[g][j] == 1 and ln[g][j] == length[g][src] and nxt[g][j] == end_id, (g, j)
            else:
                assert dn[g][j] == 0 and ln[g][j] == length[g][src] + 1 and nxt[g][j] == (key if key < V else unk_id), (g, j)
    return merged


@pytest.mark.parametrize("K", [2, 3, 8])
@pytest.mark.parametrize("V", [1, 3, 300, 20000])
def test_selection_kernels_against_restatement(V, K):
    """Step 0 from a fresh state, then a step from the kernel's own state with new logits.  V = 1 and V = 3 (< K for most K) leave slots
    empty; V = 3 also makes most candidates out-of-vocabulary copies; larger V mixes groups inside and outside T."""
    gen = torch.Generator().manual_seed(V * 10 + K)
    G = 5
    x, s, lse, origin, values, vocab = beam_case(V, G, K, gen)
    kw = {"end_id": 0, "unk_id": 0} if V == 1 else {}
    state = new_state(G, K, V)
    before = run_kernel(x, s, lse, origin, values, vocab, K, state, 0, **kw)
    check_step(x, s, lse, origin, values, vocab, K, state, before, 0, **kw)
    x2 = quantised(gen, tuple(x.shape))
    s2 = quantised(gen, tuple(s.shape), -6.0, 6.0)
    lse2 = lse_of(s2, origin, G)
    before = run_kernel(x2, s2, lse2, origin, values, vocab, K, state, 1, **kw)
    check_step(x2, s2, lse2, origin, values, vocab, K, state, before, 1, **kw)


@pytest.mark.parametrize("K", [2, 3, 8])
def test_copies_only(K):
    """V = 3 and only out-of-vocabulary copies: beyond the 3 vocabulary entries every candidate is a copy (key >= V, feeds UNK)."""
    V, G = 3, 2
    vocab = vocab_of(V)
    values = ["oa", "ob", "oc", "oa", "od", "oe", "of", "og", "oh", "oi", "oj"]
    origin = torch.tensor([0] * 11)
    x = torch.full((G * K, V), -20.0, dtype=torch.float64)
    s = torch.tensor([[1.0 + 0.25 * i + 0.125 * k for k in range(K)] for i in range(len(values))], dtype=torch.float64)
    lse = lse_of(s, origin, G)
    state = new_state(G, K, V)
    before = run_kernel(x, s, lse, origin, values, vocab, K, state, 0)
    merged = check_step(x, s, lse, origin, values, vocab, K, state, before, 0)
    assert all(e[3] >= V for e in merged[0][:K])
    assert state.next_ids.cpu()[:K].tolist() == [0] * K        # UNK


@pytest.mark.parametrize("K", [2, 3, 8])
def test_exact_ties_within_and_across_slots(K):
    """Equal inputs make exact ties: many equal logits at the K-th place inside a slot (the lower id first), and two slots with the
    same row, the same copy scores and the same total (the lower slot first)."""
    V, G = 50, 2
    vocab = vocab_of(V)
    x = torch.zeros(G * K, V, dtype=torch.float64)
    x[:, 10:30] = 1.0                   # 20 ids tied at the top of every row
    values = ["v12", "v12", "oa"]
    origin = torch.tensor([0, 0, 1])
    s = torch.full((3, K), -2.0, dtype=torch.float64)
    lse = lse_of(s, origin, G)
    state = new_state(G, K, V)
    # step 1 from a constructed state: every slot live with the same total
    set_state(state, np.full((G, K), -1.5), np.zeros((G, K)), np.zeros((G, K)), np.ones((G, K)))
    before = run_kernel(x, s, lse, origin, values, vocab, K, state, 1)
    merged = check_step(x, s, lse, origin, values, vocab, K, state, before, 1)
    # graph 0: v12's group scores above the tied ids in every slot, and the equal totals go to the lower slot first
    bp, kt = state.backpointers[1].cpu().tolist(), state.keys[1].cpu().tolist()
    assert kt[0] == [12] * K and bp[0] == list(range(K))
    # graph 1: every slot has the same candidates and the same total: slot 0's K best win, in id order
    assert bp[1] == [0] * K and kt[1] == list(range(10, 10 + K))
    assert merged[1][K - 1][0] == merged[1][K][0], "the K-th place is an exact tie"


@pytest.mark.parametrize("K", [2, 3, 8])
def test_done_slots_compete_with_live_ones(K):
    gen = torch.Generator().manual_seed(40 + K)
    V, G = 300, 4
    x, s, lse, origin, values, vocab = beam_case(V, G, K, gen)
    state = new_state(G, K, V)
    done = np.zeros((G, K))
    done[:, ::2] = 1                    # every other slot done
    total = -np.linspace(0.5, 12.0, G * K).reshape(G, K)        # descending along each graph's slots, as a merge leaves them
    set_state(state, total, done, np.zeros((G, K)), np.full((G, K), 2))
    before = run_kernel(x, s, lse, origin, values, vocab, K, state, 1)
    merged = check_step(x, s, lse, origin, values, vocab, K, state, before, 1)
    picked_done = sum(1 for g in range(G) for e in merged[g][:K] if e[3] == BR.DONE_KEY)
    picked_live = sum(1 for g in range(G) for e in merged[g][:K] if e[3] != BR.DONE_KEY)
    assert picked_done > 0 and picked_live > 0


@pytest.mark.parametrize("K", [2, 3, 8])
def test_all_slots_done_change_nothing(K):
    gen = torch.Generator().manual_seed(50 + K)
    V, G = 101, 3
    x, s, lse, origin, values, vocab = beam_case(V, G, K, gen)
    state = new_state(G, K, V)
    run_kernel(x, s, lse, origin, values, vocab, K, state, 0)
    state.done.masked_fill_(state.empty == 0, 1)
    before = state.buffer.clone()
    x2, _, _, _, _, _ = beam_case(V, G, K, gen)
    run_kernel(x2, s, lse, origin, values, vocab, K, state, 1)
    T, gk = state.max_len, G * K
    assert torch.equal(state.buffer[2 * T * gk:], before[2 * T * gk:]), "totals, lengths, done and empty flags"
    live = (state.empty == 0).cpu()
    ar = torch.arange(K).expand(G, K)
    assert torch.equal(state.backpointers[1].cpu()[live], ar[live]) and bool((state.keys[1].cpu() == -1).all())
    assert bool((state.next_ids.cpu() == 2).all())
    assert torch.equal(state.gather_idx.cpu(), torch.arange(gk))
    assert bool(torch.isnan(state.stats()).all())


def test_unsupported_beam_width_and_vocabulary_are_refused_before_any_launch():
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import decoding

    lib = N.lib()
    assert lib.ptgnn_b200_beam_select_supported(65536, 8) and not lib.ptgnn_b200_beam_select_supported(65537, 8)
    assert not lib.ptgnn_b200_beam_select_supported(100, 9) and not lib.ptgnn_b200_beam_select_supported(100, 0)
    vocab = vocab_of(20)
    module = graph2seq_module(len(vocab), 16, 32, 16)
    args = dict(input_concrete_values=["a"], input_memories=torch.zeros(1, 16, device="cuda"),
                input_memories_origin_idx=torch.zeros(1, dtype=torch.int64, device="cuda"), initial_states=torch.zeros(1, 32, device="cuda"),
                neural_model=module)
    launches = N.launch_count()
    with pytest.raises(NotImplementedError, match="beam_width"):
        decoding.beam_decode(GR.DecoderModelStub(vocab, 4), beam_width=9, **args)
    with pytest.raises(ValueError, match="beam_width"):
        decoding.beam_decode(GR.DecoderModelStub(vocab, 4), beam_width=0, **args)
    big = GR.TokenVocab([GR.UNK, GR.START, GR.END] + [f"v{i}" for i in range(65535)])
    with pytest.raises(NotImplementedError, match="65536"):
        decoding.beam_decode(GR.DecoderModelStub(big, 4), beam_width=2, **{**args, "neural_model": graph2seq_module(len(big), 16, 32, 16)})
    assert N.launch_count() == launches


# ---- the whole decode --------------------------------------------------------------------------------------------------------
def beam_decode(vocab, max_len, module, values, memories, origin, h0, K):
    from ptgnn_b200 import decoding

    return decoding.beam_decode(GR.DecoderModelStub(vocab, max_len), input_concrete_values=values, input_memories=memories.cuda(),
                                input_memories_origin_idx=origin.cuda(), initial_states=h0.cuda(), neural_model=module, beam_width=K)


def fixture_module(f):
    sd = f["sd"]
    V, E = sd["_GruCopyingDecoder__embedding_layer.weight"].shape
    H = sd["_GruCopyingDecoder__output_gru.weight_hh_l0"].shape[1]
    D = sd["_GruCopyingDecoder__memories_to_copy_attention.weight"].shape[1]
    module = graph2seq_module(V, E, H, D)
    module.load_state_dict(sd)
    return module


def assert_width_one_is_greedy(greedy, beams):
    assert len(greedy) == len(beams)
    for (tok, lp), hyps in zip(greedy, beams):
        assert len(hyps) == 1
        assert hyps[0][0] == tok and isinstance(hyps[0][1], np.float32) and hyps[0][1].tobytes() == lp.tobytes(), (tok, lp, hyps)


@pytest.mark.parametrize("name", ["greedy_small", "greedy_rank", "greedy_end"])
def test_width_one_is_greedy_on_the_fixtures(name):
    f = load(name)
    vocab = GR.TokenVocab([str(t) for t in f["vocab"]])
    module = fixture_module(f)
    T = int(f["max_seq_len"])
    values = [str(v) for v in f["values"]]
    args = (vocab, T, module, values, torch.from_numpy(f["memories"]), torch.from_numpy(f["origin"]), torch.from_numpy(f["initial_states"]))
    assert_width_one_is_greedy(native_decode(*args), beam_decode(*args, 1))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_width_one_is_greedy_at_graph2seq_shape(dtype):
    vocab, values, memories, origin, h0 = graph2seq_inputs()
    module = seeded_module()
    args = (vocab, 8, module, values, memories.to(dtype), origin, h0)
    assert_width_one_is_greedy(native_decode(*args), beam_decode(*args, 1))


def device_run(vocab, T, module, values, memories, origin, h0, K):
    from ptgnn_b200 import decoding

    dec = decoding.NativeBeamDecode(GR.DecoderModelStub(vocab, T), module, values, memories.cuda(), origin.cuda(), h0.cuda(), K)
    state = dec.run()
    return dec, state, dec.result(state)


def hypothesis_keys(tokens, values, vocab):
    keys = dict(zip(values, GR.row_keys(values, vocab)))
    return [keys[t] if t in keys else vocab.get_id_or_unk(t) for t in tokens]


def rescore(module, vocab, values, memories, origin, h0, hyps, T):
    """Each hypothesis (graph, key list) scored on its own by teacher forcing through the restatement's dictionary rule: the sum over
    its steps of the dictionary score of its key there (END at the step it ends, when shorter than T)."""
    sd = {k: v.detach().cpu().double() for k, v in module.state_dict().items()}
    V = len(vocab)
    keys = GR.row_keys(values, vocab)
    end_id, unk_id, start_id = vocab.get_id_or_unk(GR.END), vocab.get_id_or_unk(GR.UNK), vocab.get_id_or_unk(GR.START)
    n = len(hyps)
    graphs = torch.tensor([g for g, _ in hyps])
    seqs = [p + [end_id] if len(p) < T else p for _, p in hyps]
    # the memories of each hypothesis's graph, as a graph of its own
    rows = [np.flatnonzero(origin.numpy() == g) for g, _ in hyps]
    mem = torch.cat([memories.double()[r] for r in rows])
    org = torch.cat([torch.full((len(r),), i, dtype=torch.int64) for i, r in enumerate(rows)])
    row_keys = [keys[i] for r in rows for i in r]
    h = h0.double()[graphs]
    ids = [start_id] * n
    scores = [0.0] * n
    with torch.no_grad():
        for t in range(T):
            copy_lp, target_lp, h_new = DR_compute(sd, h, mem, org, ids)
            h = h_new
            lp, c = target_lp.numpy(), copy_lp.numpy()
            for i in range(n):
                if t >= len(seqs[i]):
                    continue
                entries = dict(BR.dictionary(lp[i], c, np.flatnonzero(org.numpy() == i), row_keys))
                scores[i] += entries.get(seqs[i][t], -math.inf)
            ids = [end_id if t >= len(seqs[i]) else seqs[i][t] if seqs[i][t] < V else unk_id for i in range(n)]
    return scores


def DR_compute(sd, h, mem, org, ids):
    import decoder_reference as DR

    copy_lp, target_lp, h_new = DR.compute_logprobs(sd, h, mem, org, torch.tensor(ids)[:, None])
    return copy_lp[:, 0], target_lp[:, 0], h_new[0]


@pytest.mark.parametrize("K", [2, 4, 5, 8])
def test_graph2seq_shape_against_restatement(K):
    vocab, values, memories, origin, h0 = graph2seq_inputs(G=20 if K == 8 else 30)
    module = seeded_module()
    T = 8
    G, V, M = h0.shape[0], len(vocab), origin.numel()
    dec, state, out = device_run(vocab, T, module, values, memories, origin, h0, K)
    _, _, again = device_run(vocab, T, module, values, memories, origin, h0, K)
    assert [[(t, lp.tobytes()) for t, lp in hs] for hs in again] == [[(t, lp.tobytes()) for t, lp in hs] for hs in out], "two runs differ"

    # sorted and distinct per graph
    for hs in out:
        totals = [float(lp) for _, lp in hs]
        assert totals == sorted(totals, reverse=True)
        assert len({tuple(t) for t, _ in hs}) == len(hs)

    # the restatement driven along the device's choices
    bp, kt = state.backpointers.cpu().numpy(), state.keys.cpu().numpy()
    empty_final = state.empty.cpu().numpy()
    sd = {k: v.detach().cpu().double() for k, v in module.state_dict().items()}
    keys = GR.row_keys(values, vocab)
    end_id, unk_id, start_id = vocab.get_id_or_unk(GR.END), vocab.get_id_or_unk(GR.UNK), vocab.get_id_or_unk(GR.START)
    mem_rep, org_rep = BR.replicate(memories.double(), origin, K)
    h = h0.double().repeat_interleave(K, 0)
    ids = [start_id] * (G * K)
    status = [[BR.LIVE if k == 0 else BR.EMPTY for k in range(K)] for _ in range(G)]
    cum = [[0.0] * K for _ in range(G)]
    clear = live_steps = 0
    with torch.no_grad():
        for t in range(T):
            lp, c, h_new = BR.compute_logprobs_beams(sd, h, mem_rep, org_rep, ids, M, K)
            new_status = [[BR.EMPTY] * K for _ in range(G)]
            new_cum = [[0.0] * K for _ in range(G)]
            gather = []
            for g in range(G):
                rows = np.flatnonzero(origin.numpy() == g)
                cands = [BR.slot_candidates(status[g][k], cum[g][k], lp[g * K + k], c[k], rows, keys, K) for k in range(K)]
                m = BR.merge(cands, K)
                got = {(int(bp[t, g, j]), int(kt[t, g, j])) for j in range(K) if bp[t, g, j] >= 0}
                if any(st == BR.LIVE for st in status[g]):
                    live_steps += 1
                    bound = STEP_BOUND * (t + 1) * (1 + abs(m[min(K, len(m)) - 1][0]))
                    if len(m) <= K or m[K - 1][0] - m[K][0] > bound:
                        assert got == {(e[1], e[3]) for e in m[:K]}, f"graph {g} step {t}"
                        clear += 1
                for j in range(K):
                    p, key = int(bp[t, g, j]), int(kt[t, g, j])
                    gather.append(g * K + (p if p >= 0 else j))
                    if p < 0:
                        continue
                    entry = [e for e in m if (e[1], e[3]) == (p, key)]
                    if entry:
                        new_cum[g][j] = entry[0][0]
                    else:                   # outside the restatement's K best of its slot: its dictionary score there
                        d = dict(BR.dictionary(lp[g * K + p], c[p], rows, keys))
                        new_cum[g][j] = cum[g][p] + d[key]
                    new_status[g][j] = BR.DONE if key == BR.DONE_KEY or key == end_id else BR.LIVE
            status, cum = new_status, new_cum
            h = h_new[gather]
            ids = []
            for g in range(G):
                for j in range(K):
                    key = int(kt[t, g, j])
                    ids.append(end_id if key < 0 or key == end_id else key if key < V else unk_id)
    assert clear >= 0.9 * live_steps, (clear, live_steps)
    for g in range(G):
        for j, (tok, lp) in enumerate(out[g]):
            assert not empty_final[g, j]
            assert abs(float(lp) - cum[g][j]) <= STEP_BOUND * T * (1 + abs(cum[g][j])), (g, j, float(lp), cum[g][j])

    # every returned hypothesis re-scored on its own
    hyps = [(g, hypothesis_keys(tok, values, vocab)) for g in range(G) for tok, _ in out[g]]
    scores = rescore(module, vocab, values, memories, origin, h0, hyps, T)
    flat = [lp for g in range(G) for _, lp in out[g]]
    for (g, p), score, lp in zip(hyps, scores, flat):
        assert abs(float(lp) - score) <= STEP_BOUND * T * (1 + abs(score)), (g, p, float(lp), score)


def test_decode_loop_has_no_host_synchronisation_and_a_constant_launch_count():
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import decoding

    vocab, values, memories, origin, h0 = graph2seq_inputs(seed=9, G=20)
    module = seeded_module()
    mem, org, h = memories.cuda(), origin.cuda(), h0.cuda()
    per_step = {}
    for K in (1, 2, 3, 8):
        counts = []
        for T in (1, 2, 3, 5):              # the first run also builds the graph plan (cached afterwards)
            dec = decoding.NativeBeamDecode(GR.DecoderModelStub(vocab, T), module, values, mem, org, h, K)
            torch.cuda.synchronize()
            before = N.launch_count()
            torch.cuda.set_sync_debug_mode("error")
            try:
                state = dec.run()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            counts.append(N.launch_count() - before)
            dec.result(state)
        per_step[K] = counts[2] - counts[1]
        assert per_step[K] > 0 and counts[3] - counts[2] == 2 * per_step[K], (K, counts)
    assert len(set(per_step.values())) == 1, per_step
