"""graph2seq greedy decoding on the GPU: the selection kernel element by element against the float64 restatement
(greedy_decode_reference.py), the whole native decode against the reference's fixtures, at graph2seq's shape against the restatement
driven step by step, bf16 memories against fp32, bit-identical reruns, no host synchronisation in the decode loop, a constant launch
count per step, and the refusals.

Bounds, u = 2^-24, gamma_k = k u / (1 - k u).  Z is a strided per-thread sum of V / 1024 terms, a 10-level tree and one more term, each
term expf(x - max) with a relative error of at most 2 u + u |x - max| e^(x - max) <= 3 u: |dZ| <= B_Z = gamma_{ceil(V / 1024) + 11}
+ 3 u + u (|log S| + |Z|) with S the sum.  A score is lp = fl(x - Z) (|dZ| + u |lp|), merged with n copy terms fl(s - Z) by n float32
logaddexps (each <= 4 u (1 + |result|)): |dscore| <= B_Z + (1 + 5 n) u (1 + |score|).  Both are checked with a factor 2 of slack.  A
whole decode step adds the fp32 rounding of the GRU, the two attentions and the vocabulary projection: 2e-5 (1 + |score|) per step.
"""
import math
import os

import numpy as np
import pytest
import torch

import greedy_decode_reference as GR

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STEP_BOUND = 2e-5


def gamma(k):
    return k * U / (1 - k * U)


def vocab_of(V):
    if V == 1:
        return GR.TokenVocab([GR.UNK])
    return GR.TokenVocab([GR.UNK, GR.START, GR.END] + [f"v{i}" for i in range(3, V)])


def quantised(gen, shape, lo=-8.0, hi=8.0, step=1 / 64):
    """Values on a 1/64 grid: x - Z stays exact enough that distinct values keep distinct fp32 keys, and ties are exact."""
    n = int((hi - lo) / step)
    return torch.randint(0, n, shape, generator=gen).double() * step + lo


def run_kernel(x, s, lse, origin, values, vocab, state=None, step=0, end_id=2, unk_id=0, max_len=4):
    """One ptgnn_b200_decode_select call on fresh (or the given) state; returns the state and the [G, 2] (Z, score) record."""
    from ptgnn_b200 import decoding

    G, V = x.shape
    groups = decoding.CopyGroups(values, origin.numpy(), G, vocab)
    if state is None:
        state = decoding.DecodeState(G, max_len, V, 1 if V > 1 else 0, "cuda")
    decoding.decode_select(x.float().cuda(), s.float().cuda(), lse.float().cuda(), groups.to_device("cuda"), state, step, end_id, unk_id)
    return state, state.stats().cpu().double()


def case(V, G, gen, copies_per_graph=12):
    """Logits [G, V] (ties everywhere for large V), copy scores with their graphs' lse, and values mixing vocabulary tokens inside and
    outside the top 100, the top-1 token, and out-of-vocabulary strings repeated within a graph; graph G - 1 has no memories."""
    vocab = vocab_of(V)
    x = quantised(gen, (G, V))
    origin, values = [], []
    for g in range(G - 1):
        order = np.lexsort((np.arange(V), -x[g].numpy()))
        picks = [int(order[0]), int(order[min(99, V - 1)]), int(order[min(100, V - 1)]), int(order[-1])]
        for j in range(copies_per_graph):
            r = int(torch.randint(0, 6, (1,), generator=gen))
            if r < 4 and V > 3:
                tok = picks[r] if picks[r] >= 3 else 3 + picks[r] % max(1, V - 3)
                values.append(vocab.get_name_for_id(min(tok, V - 1)))
            else:
                values.append(f"oov{int(torch.randint(0, 5, (1,), generator=gen))}")
            origin.append(g)
    origin = torch.tensor(origin, dtype=torch.int64)
    perm = torch.randperm(len(values), generator=gen)
    origin, values = origin[perm], [values[int(i)] for i in perm]
    s = quantised(gen, (len(values),), -6.0, 6.0)
    s32 = s.float().double()
    lse = torch.full((G,), -math.inf, dtype=torch.float64)
    for g in range(G):
        if (origin == g).any():
            lse[g] = torch.logsumexp(s32[origin == g], 0)
    return x, s, lse.float().double(), origin, values, vocab


def bounds(x, Z, score, n_members):
    V = x.shape[1]
    m = x.max(dim=1).values
    logS = (Z - m).abs()
    bz = gamma(math.ceil(V / 1024) + 11) + 3 * U + U * (logS + Z.abs())
    return 2 * bz, 2 * (bz + (1 + 5 * n_members) * U * (1 + score.abs()))


def check_step(x, s, lse, origin, values, vocab, state, stats, prev=None, end_id=2, unk_id=0):
    """The kernel's state and (Z, score) against the restatement; prev: ((tokens, logprobs, done) before the step, the log-probability
    bounds so far).  Returns the same pair after the step."""
    G, V = x.shape
    keys = GR.row_keys(values, vocab)
    Z, picks = GR.select_from_logits(x.numpy(), s.numpy(), lse.numpy(), origin.numpy(), keys)
    Z = torch.from_numpy(Z)
    (tokens, logprobs, done), err = prev if prev is not None else (([[] for _ in range(G)], [0.0] * G, [False] * G), [0.0] * G)
    live = [g for g in range(G) if not done[g]]
    n = torch.tensor([sum(1 for i in range(len(keys)) if origin[i] == g and keys[i] == picks[g][0]) for g in range(G)], dtype=torch.float64)
    bz, bs = bounds(x, Z, torch.tensor([p[1] for p in picks]), n)
    got_len, got_done = state.length.cpu().tolist(), state.done.cpu().tolist()
    got_tok = state.tokens.cpu().tolist()
    for g in live:
        assert abs(stats[g, 0].item() - Z[g].item()) <= bz[g].item(), f"graph {g}: Z {stats[g, 0].item()} vs {Z[g].item()} (bound {bz[g]:.2e})"
        assert abs(stats[g, 1].item() - picks[g][1]) <= bs[g].item(), f"graph {g}: score {stats[g, 1].item()} vs {picks[g][1]}"
        if not (picks[g][2] > bs[g].item() or picks[g][2] == 0.0):
            # a near tie (margin within the bound): the kernel may take any entry within the bound of the best; follow its pick
            got = end_id if got_done[g] else got_tok[g][got_len[g] - 1]
            entries = picks[g][3]
            assert got in entries and picks[g][1] - entries[got] <= bs[g].item(), f"graph {g}: pick {got} outside the near tie"
            picks[g] = (got, entries[got], picks[g][2], entries)
    ref_state = ([list(t) for t in tokens], list(logprobs), list(done))
    nxt = GR.update(ref_state, picks, end_id, unk_id, V)
    assert [bool(d) for d in state.done.cpu().tolist()] == ref_state[2]
    assert got_len == [len(t) for t in ref_state[0]]
    assert [got_tok[g][:got_len[g]] for g in range(G)] == ref_state[0]
    assert state.next_ids.cpu().tolist() == nxt
    lp = state.logprob.cpu().double()
    err = [err[g] + (bs[g].item() + U * abs(ref_state[1][g]) if g in live else 0.0) for g in range(G)]
    for g in range(G):
        assert abs(lp[g].item() - ref_state[1][g]) <= err[g], f"graph {g}: logprob {lp[g].item()} vs {ref_state[1][g]}"
    return ref_state, err


@pytest.mark.parametrize("V", [1, 99, 100, 101, 20000, 65536])
def test_selection_kernel_against_restatement(V):
    gen = torch.Generator().manual_seed(V)
    G = 7
    x, s, lse, origin, values, vocab = case(V, G, gen)
    if V == 1:
        state, stats = run_kernel(x, s, lse, origin, values, vocab, end_id=0, unk_id=0)
        check_step(x, s, lse, origin, values, vocab, state, stats, end_id=0, unk_id=0)
        return
    state, stats = run_kernel(x, s, lse, origin, values, vocab)
    prev = check_step(x, s, lse, origin, values, vocab, state, stats)
    # a second step on the same state with new logits and copy scores
    x2 = quantised(gen, (G, V))
    s2 = quantised(gen, (len(values),), -6.0, 6.0)
    lse2 = torch.tensor([torch.logsumexp(s2.float().double()[origin == g], 0).item() if (origin == g).any() else -math.inf for g in range(G)])
    state, stats = run_kernel(x2, s2, lse2.float().double(), origin, values, vocab, state=state, step=1)
    check_step(x2, s2, lse2.float().double(), origin, values, vocab, state, stats, prev=prev)


def test_exact_ties_at_the_kth_value_and_the_top_1():
    """Logits of few distinct values: the 100th value is tied many times over, and so is the maximum.  Copies of tied ids on both sides
    of the cut decide whether their vocabulary mass is merged (lower ids are in T).  Without copies the lowest maximal id wins."""
    V, G = 1000, 4
    vocab = vocab_of(V)
    x = torch.zeros(G, V, dtype=torch.float64)
    x[:, 3::7] = 1.0                       # 143 ids at the top: T takes the 100 lowest of them
    x[:, 500:] -= 2.0
    order = np.lexsort((np.arange(V), -x[0].numpy()))
    inside, outside = int(order[99]), int(order[100])
    assert x[0, inside] == x[0, outside]
    values = [vocab.get_name_for_id(inside)] * 3 + [vocab.get_name_for_id(outside)] * 3 + [vocab.get_name_for_id(outside)] * 3
    origin = torch.tensor([0, 0, 0, 1, 1, 1, 2, 2, 2])
    s = torch.zeros(len(values), dtype=torch.float64)
    lse = torch.tensor([math.log(3)] * 3 + [-math.inf], dtype=torch.float64)
    state, stats = run_kernel(x, s, lse, origin, values, vocab)
    check_step(x, s, lse, origin, values, vocab, state, stats)
    # graph 0's copies merge with their in-T entry; graph 1's do not; graph 3 has no copies and picks the lowest maximal id
    assert state.tokens[0, 0].item() == inside and state.tokens[1, 0].item() == outside
    assert state.tokens[3, 0].item() == int(order[0]) == 3


def test_copy_of_the_top_1_and_every_group_outside_t():
    V, G = 300, 3
    gen = torch.Generator().manual_seed(3)
    vocab = vocab_of(V)
    x = quantised(gen, (G, V))
    order = [np.lexsort((np.arange(V), -x[g].numpy())) for g in range(G)]
    top = int(order[0][0])
    low = [vocab.get_name_for_id(int(v)) for v in order[1][::-1] if v >= 3][:3]     # the lowest-ranked ids other than UNK, START, END
    # graph 0: a copy of its top-1 token; graph 1: vocabulary copies all outside T and out-of-vocabulary ones, two groups exactly tied
    values = [vocab.get_name_for_id(top), "zz", "zz"] + low + ["oa", "ob"]
    origin = torch.tensor([0, 0, 0, 1, 1, 1, 1, 1])
    s = torch.tensor([-4.0, -9.0, -9.0, 30.0, 30.0, 29.0, 30.0, 30.0], dtype=torch.float64)
    lse = torch.tensor([torch.logsumexp(s[origin == g], 0).item() if (origin == g).any() else -math.inf for g in range(G)])
    state, stats = run_kernel(x, s, lse, origin, values, vocab)
    check_step(x, s, lse, origin, values, vocab, state, stats)
    assert state.tokens[0, 0].item() == top
    assert state.tokens[1, 0].item() == vocab.get_id_or_unk(low[0]), "equal scores: the first group in first-occurrence order"
    assert state.next_ids[1].item() == vocab.get_id_or_unk(low[0])


def test_all_graphs_already_done_change_nothing():
    V, G = 101, 4
    gen = torch.Generator().manual_seed(4)
    x, s, lse, origin, values, vocab = case(V, G, gen)
    state, _ = run_kernel(x, s, lse, origin, values, vocab)
    state.done.fill_(1)
    before = state.buffer.clone()
    state, stats = run_kernel(x, s, lse, origin, values, vocab, state=state, step=1)
    assert torch.equal(state.buffer, before)
    assert state.next_ids.cpu().tolist() == [2] * G
    assert bool(torch.isnan(stats).all())


def test_unsupported_vocabulary_is_refused_before_any_launch():
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import decoding

    assert N.lib().ptgnn_b200_decode_select_supported(65536) and not N.lib().ptgnn_b200_decode_select_supported(65537)
    assert not N.lib().ptgnn_b200_decode_select_supported(0)
    launches = N.launch_count()
    with pytest.raises(NotImplementedError, match="65536"):
        decoding.check_vocab_size(65537)
    vocab = GR.TokenVocab([GR.UNK, GR.START, GR.END] + [f"v{i}" for i in range(65535)])
    module = graph2seq_module(len(vocab), 16, 32, 16)
    with pytest.raises(NotImplementedError, match="65536"):
        decoding.greedy_decode(GR.DecoderModelStub(vocab, 4), input_concrete_values=["a"], input_memories=torch.zeros(1, 16, device="cuda"),
                               input_memories_origin_idx=torch.zeros(1, dtype=torch.int64, device="cuda"),
                               initial_states=torch.zeros(1, 32, device="cuda"), neural_model=module)
    assert N.launch_count() == launches


# ---- the whole decode --------------------------------------------------------------------------------------------------------
def graph2seq_module(V, E, H, D, seed=0):
    import ptgnn_b200 as P

    torch.manual_seed(seed)
    return P.GruCopyingDecoder(V, E, H, D, unk_id=0, dropout_rate=0.2).cuda().eval()


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    f = {k: z[k] for k in z.files}
    f["sd"] = {k[4:]: torch.from_numpy(v) for k, v in f.items() if k.startswith("sd::")}
    ends = np.cumsum(f["out_lengths"])
    f["ref_tokens"] = [[str(t) for t in f["out_tokens"][e - n:e]] for e, n in zip(ends, f["out_lengths"])]
    return f


def native_decode(vocab, max_len, module, values, memories, origin, h0):
    from ptgnn_b200 import decoding

    return decoding.greedy_decode(GR.DecoderModelStub(vocab, max_len), input_concrete_values=values, input_memories=memories.cuda(),
                                  input_memories_origin_idx=origin.cuda(), initial_states=h0.cuda(), neural_model=module)


@pytest.mark.parametrize("name", ["greedy_small", "greedy_rank", "greedy_end"])
def test_whole_decode_matches_reference_fixture(name):
    f = load(name)
    vocab = GR.TokenVocab([str(t) for t in f["vocab"]])
    sd = f["sd"]
    V, E = sd["_GruCopyingDecoder__embedding_layer.weight"].shape
    H = sd["_GruCopyingDecoder__output_gru.weight_hh_l0"].shape[1]
    D = sd["_GruCopyingDecoder__memories_to_copy_attention.weight"].shape[1]
    module = graph2seq_module(V, E, H, D)
    module.load_state_dict(sd)
    T = int(f["max_seq_len"])
    values = [str(v) for v in f["values"]]
    out = native_decode(vocab, T, module, values, torch.from_numpy(f["memories"]), torch.from_numpy(f["origin"]),
                        torch.from_numpy(f["initial_states"]))
    assert [t for t, _ in out] == f["ref_tokens"]
    for (_, lp), ref in zip(out, f["out_logprobs"]):
        assert isinstance(lp, np.float32)
        assert abs(float(lp) - float(ref)) <= STEP_BOUND * T * (1 + abs(float(ref))), (name, lp, ref)
    again = native_decode(vocab, T, module, values, torch.from_numpy(f["memories"]), torch.from_numpy(f["origin"]),
                          torch.from_numpy(f["initial_states"]))
    assert [(t, lp.tobytes()) for t, lp in again] == [(t, lp.tobytes()) for t, lp in out]


def graph2seq_inputs(seed=5, G=50, D=128, V=20000):
    gen = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, 60, (G,), generator=gen)
    counts[7] = 0
    origin = torch.repeat_interleave(torch.arange(G), counts)
    origin = origin[torch.randperm(origin.numel(), generator=gen)]
    vocab = vocab_of(V)
    values = [f"v{int(i)}" if i < V else f"ident{int(i) - V}" for i in torch.randint(3, V + 400, (origin.numel(),), generator=gen)]
    memories = torch.randn(origin.numel(), D, generator=gen)
    h0 = torch.randn(G, 128, generator=gen)
    return vocab, values, memories, origin, h0


def seeded_module(V=20000, E=256, H=128, D=128):
    module = graph2seq_module(V, E, H, D, seed=6)
    with torch.no_grad():
        module._GruCopyingDecoder__vocab_bias.normal_(0.0, 2.0, generator=torch.Generator(device="cuda").manual_seed(7))
    return module


def picks_of(out, vocab, values, T):
    """Each graph's key at each step, from a decode's result (END at the step it ends, None afterwards)."""
    V = len(vocab)
    keys = dict(zip(values, GR.row_keys(values, vocab)))
    end_id = vocab.get_id_or_unk(GR.END)
    res = []
    for toks, _ in out:
        p = [keys[t] if t in keys else vocab.get_id_or_unk(t) for t in toks]
        if len(p) < T:
            p.append(end_id)
        res.append(p + [None] * (T - len(p)))
    return res


def restated_along(module, vocab, values, memories, origin, h0, picks, T):
    """The restatement driven by the given picks: per step and graph (its pick, its score of the given pick, its margin)."""
    sd = {k: v.detach().cpu().double() for k, v in module.state_dict().items()}
    memories, h = memories.double(), h0.double()
    V, G = len(vocab), h0.shape[0]
    keys = GR.row_keys(values, vocab)
    end_id, unk_id = vocab.get_id_or_unk(GR.END), vocab.get_id_or_unk(GR.UNK)
    import decoder_reference as DR

    ids = [vocab.get_id_or_unk(GR.START)] * G
    rows = []
    with torch.no_grad():
        for t in range(T):
            copy_lp, target_lp, h_new = DR.compute_logprobs(sd, h, memories, origin, torch.tensor(ids)[:, None])
            h = h_new[0]
            lp, c = target_lp[:, 0].numpy(), copy_lp[:, 0].numpy()
            sel = GR.select(lp, c, origin.numpy(), keys)
            step = []
            for g in range(G):
                k = picks[g][t]
                if k is None:
                    step.append(None)
                    continue
                if k == sel[g][0]:
                    score = sel[g][1]
                else:                   # the restatement's dictionary entry of the native pick
                    in_t = k < V and k in set(np.lexsort((np.arange(V), -lp[g]))[:min(100, V)].tolist())
                    score = float(lp[g, k]) if in_t else -math.inf
                    for i in np.flatnonzero(origin.numpy() == g):
                        if keys[i] == k:
                            score = GR.logaddexp(score, float(c[i]))
                step.append((sel[g][0], score, sel[g][2]))
            rows.append(step)
            ids = [end_id if picks[g][t] is None else picks[g][t] if picks[g][t] < V else unk_id for g in range(G)]
    return rows


def test_graph2seq_shape_against_restatement_and_bitwise_rerun():
    vocab, values, memories, origin, h0 = graph2seq_inputs()
    module = seeded_module()
    T = 8
    out = native_decode(vocab, T, module, values, memories, origin, h0)
    again = native_decode(vocab, T, module, values, memories, origin, h0)
    assert [(t, lp.tobytes()) for t, lp in again] == [(t, lp.tobytes()) for t, lp in out], "two runs differ"
    picks = picks_of(out, vocab, values, T)
    rows = restated_along(module, vocab, values, memories, origin, h0, picks, T)
    clear = 0
    for g in range(len(out)):
        total = 0.0
        for t in range(T):
            r = rows[t][g]
            if r is None:
                break
            want, score, margin = r
            total += score
            if margin > STEP_BOUND * (1 + abs(score)):
                assert picks[g][t] == want, f"graph {g} step {t}: native {picks[g][t]} vs restatement {want} (margin {margin:.2e})"
                clear += 1
        assert abs(float(out[g][1]) - total) <= STEP_BOUND * T * (1 + abs(total)), (g, out[g][1], total)
    assert clear >= 0.9 * sum(1 for t in range(T) for g in range(len(out)) if rows[t][g] is not None)


def test_bf16_memories_against_fp32_on_clear_margin_steps():
    vocab, values, memories, origin, h0 = graph2seq_inputs(seed=8)
    module = seeded_module()
    T = 8
    mb = memories.to(torch.bfloat16)
    out32 = native_decode(vocab, T, module, values, mb.float(), origin, h0)
    out16 = native_decode(vocab, T, module, values, mb, origin, h0)
    p32, p16 = picks_of(out32, vocab, values, T), picks_of(out16, vocab, values, T)
    rows = restated_along(module, vocab, values, mb.float(), origin, h0, p32, T)
    compared = 0
    for g in range(len(out32)):
        for t in range(T):
            r = rows[t][g]
            if r is None or r[2] <= 0.05:        # bf16 A and C move the logits by ~2^-8 relative: stop at the first close call
                break
            assert p16[g][t] == p32[g][t], f"graph {g} step {t}"
            compared += 1
    assert compared >= 100


def test_decode_loop_has_no_host_synchronisation_and_a_constant_launch_count():
    from ptgnn_b200 import _native as N
    from ptgnn_b200 import decoding

    vocab, values, memories, origin, h0 = graph2seq_inputs(seed=9, G=20)
    module = seeded_module()
    mem, org, h = memories.cuda(), origin.cuda(), h0.cuda()
    counts = []
    for T in (1, 2, 3, 5):                  # the first run also builds the graph plan (cached afterwards)
        dec = decoding.NativeGreedyDecode(GR.DecoderModelStub(vocab, T), module, values, mem, org, h)
        torch.cuda.synchronize()
        before = N.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            state = dec.run()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        counts.append(N.launch_count() - before)
        dec.result(state)
    per_step = counts[2] - counts[1]
    assert per_step > 0 and counts[3] - counts[2] == 2 * per_step, counts
