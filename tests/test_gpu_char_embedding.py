"""GPU tests of the native CharUnitEmbedder (csrc/char_cnn.cu, DESIGN.md §3.13): the kernel element by element against float64 under
the bound of tests/char_embedding_reference.py, the module against the reference's fixtures, bf16 under autocast, the chunked backward,
the status word, CUDA-graph capture, memory, save / restore, and two training steps."""
import copy
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import char_embedding_reference as R  # noqa: E402
from helpers import load_golden  # noqa: E402

from ptgnn_b200 import autograd as AG  # noqa: E402
from ptgnn_b200.embeddings import CharUnitEmbedder, CnnConfig  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
DEFAULT = CnnConfig(256, 3, 128, 3, 3)
T_DEFAULT = 9          # tokens per tile at L1 = 13 (two warpgroups: 128 rows)


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def module(C, D, cfg, seed=0):
    torch.manual_seed(seed)
    return CharUnitEmbedder(C, D, cfg, 0.0).to(DEV).eval()


def params(m):
    return [p.detach() for p in m._params()]


def check_forward(m, chars, bf16=False):
    with torch.no_grad():
        if bf16:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = m(chars)
            assert out.dtype == torch.bfloat16
        else:
            out = m(chars)
            assert out.dtype == torch.float32
    torch.cuda.synchronize()
    ps = params(m)
    exact = R.forward(chars, *ps)
    b = R.bound(chars, *ps, bf16=bf16)
    err = (out.double() - exact).abs()
    bad = err > b
    assert not bool(bad.any()), f"{int(bad.sum())} elements outside the bound; worst excess {float((err - b).max()):.3e}"
    if out.numel():                # the element bound is a worst case: the whole output is also held to the tighter rel. L2 bars
        if bf16:
            assert R.rel_l2(out, R.emulate_bf16(chars, *ps)) <= R.BF16_EMU_REL_L2
            assert R.rel_l2(out, exact) <= 1e-2
        else:
            assert R.rel_l2(out, exact) <= R.FP32_REL_L2
    return out


SHAPES = [   # (C, cfg, D, B, L, id pattern)
    *[(101, DEFAULT, D, 300, 15, "random") for D in (1, 63, 64, 127, 128, 256)],
    *[(101, DEFAULT, 127, B, 15, "random") for B in (0, 1, T_DEFAULT - 1, T_DEFAULT, T_DEFAULT + 1)],
    (101, DEFAULT, 63, 80_000, 15, "random"),
    (101, DEFAULT, 127, 80_000, 15, "random"),
    (101, DEFAULT, 127, 257, 7, "random"),
    (101, DEFAULT, 127, 257, 32, "random"),
    (40, CnnConfig(64, 1, 256, 5, 2), 63, 333, 12, "random"),
    (101, CnnConfig(128, 2, 64, 4, 5), 100, 333, 20, "random"),
    (101, CnnConfig(256, 3, 256, 3, 3), 256, 200, 15, "random"),
    (101, CnnConfig(64, 5, 64, 5, 5), 17, 200, 13, "random"),
    (1, DEFAULT, 64, 100, 15, "random"),
    (101, DEFAULT, 127, 100, 15, "equal"),
]


@pytest.mark.parametrize("C,cfg,D,B,L,ids", SHAPES)
def test_forward_against_float64(C, cfg, D, B, L, ids):
    m = module(C, D, cfg, seed=B + D)
    g = torch.Generator(device=DEV).manual_seed(B + L)
    chars = torch.randint(0, C, (B, L), device=DEV, generator=g) if ids == "random" else torch.full((B, L), 7, device=DEV)
    out = check_forward(m, chars)
    assert out.shape == (B, D)


@pytest.mark.parametrize("cfg,D,L", [(DEFAULT, 127, 15), (CnnConfig(64, 1, 256, 5, 2), 63, 12)])
def test_bf16_forward_against_float64(cfg, D, L):
    m = module(101, D, cfg, seed=3)
    chars = torch.randint(0, 101, (500, L), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    check_forward(m, chars, bf16=True)


def fixture_module(g, D=None):
    C, cfg, D = int(g["num_chars"]), CnnConfig(*[int(x) for x in g["cnn"]]), int(g["dim"]) if D is None else D
    m = CharUnitEmbedder(C, D, cfg, 0.2)
    w1, b1, w2, b2, w3 = R.params_of(g, D)
    sd = {R.PRE + "conv_l1.weight": w1, R.PRE + "conv_l1.bias": b1, R.PRE + "conv_l2.weight": w2, R.PRE + "conv_l2.bias": b2,
          R.PRE + "conv_l3.weight": w3}
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval()


def close(out, ref):
    ref = torch.from_numpy(np.asarray(ref)).to(DEV).double()
    assert bool(((out.double() - ref).abs() <= 1e-5 * ref.abs().clamp(min=1.0)).all()), float((out.double() - ref).abs().max())


@pytest.mark.parametrize("D", [63, 127, 128])
def test_module_matches_default_fixture(D):
    g = load_golden("char_default")
    chars = torch.from_numpy(g["chars"]).to(DEV)
    m = fixture_module(g, D)
    with torch.no_grad():
        close(m(chars), g[f"out_d{D}"])
        if D == 128:
            close(m(chars[:, :7].contiguous()), g["out_minl"])


@pytest.mark.parametrize("name", ["char_cfg_a", "char_cfg_b"])
def test_module_matches_config_fixtures(name):
    g = load_golden(name)
    m = fixture_module(g)
    with torch.no_grad():
        close(m(torch.from_numpy(g["chars"]).to(DEV)), g["out"])


def test_bf16_matches_autocast_fixture():
    g = load_golden("char_default")
    chars = torch.from_numpy(g["chars"]).to(DEV)
    m = fixture_module(g, 127)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(chars)
    ac = torch.from_numpy(g["out_bf16ac_d127"]).to(DEV)
    bars = R.n2_bars(out, ac, torch.from_numpy(g["out_d127"]).to(DEV))
    assert all(bars.values()), bars
    assert R.rel_l2(out, ac) <= R.BF16_EMU_REL_L2


def test_max_position_at_token_edges():
    """Tokens alternate between a character with large and one with small activations: pooling one row past a token's last valid
    position, or dropping a tile's last partial token, shows up as a wrong element."""
    m = module(4, 64, DEFAULT, seed=11)
    with torch.no_grad():
        w1 = m._params()[0]
        w1[:, 1] *= 30.0           # char 1: large activations
        w1[:, 2] *= 0.01           # char 2: small ones
    B, L = 4 * T_DEFAULT + 3, 15
    chars = torch.full((B, L), 2, device=DEV)
    chars[0::2] = 1
    chars[1::2, 0] = 1             # a small token whose only large character is its first one: covered by position 0 only
    out = check_forward(m, chars)
    out2 = check_forward(m, chars.flip(0))
    assert torch.equal(out.flip(0), out2)


def make_grad_case(B, seed=1):
    m = module(101, 127, CnnConfig(128, 2, 64, 4, 5), seed=seed).train()
    chars = torch.randint(0, 101, (B, 20), device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    grad_out = torch.randn(B, 127, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + 1))
    return m, chars, grad_out


def native_grads(m, chars, grad_out):
    for p in m.parameters():
        p.grad = None
    out = m(chars)
    (out * grad_out).sum().backward()
    return [p.grad.clone() for p in m._params()]


def kernel_decisions(m, chars):
    """The kernel's ReLU masks ([B, F, L] layout) and max positions, for R.gradients."""
    from ptgnn_b200 import embeddings as E

    shape = E.char_cnn_shape(m._CharUnitEmbedder__conv_l1, m._CharUnitEmbedder__conv_l2, m._CharUnitEmbedder__conv_l3)
    prepared = E.char_cnn_prepare(shape, *params(m), False, None)
    a1, a2 = E.native_char_cnn_materialise(chars, shape, prepared)
    _, arg = E.native_char_cnn(chars, shape, prepared, want_arg=True)
    B = chars.shape[0]
    m1 = (a1.view(B, -1, shape[1]) > 0).transpose(1, 2).double()
    m2 = (a2.view(B, -1, shape[3]) > 0).transpose(1, 2).double()
    return m1, m2, arg


def check_grads(m, chars, grad_out, grads):
    exact = R.gradients(chars, *params(m), grad_out, kernel_decisions(m, chars))
    for gn, ge in zip(grads, exact):
        tol = 1e-4 * ge.abs().max().clamp(min=1.0)
        assert float((gn.double() - ge).abs().max()) <= tol


def test_gradients_against_float64():
    m, chars, grad_out = make_grad_case(3000)
    check_grads(m, chars, grad_out, native_grads(m, chars, grad_out))


def test_chunked_gradients_are_bit_identical(monkeypatch):
    monkeypatch.setattr(AG, "CHAR_BACKWARD_CHUNK", 1000)
    m, chars, grad_out = make_grad_case(3001, seed=2)      # four chunks, the last of one token
    g1 = native_grads(m, chars, grad_out)
    g2 = native_grads(m, chars, grad_out)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    check_grads(m, chars, grad_out, g1)
    monkeypatch.setattr(AG, "CHAR_BACKWARD_CHUNK", 4096)
    g3 = native_grads(m, chars, grad_out)
    check_grads(m, chars, grad_out, g3)


def test_gradients_match_fixture():
    g = load_golden("char_cfg_b")
    m = fixture_module(g).train()
    m._CharUnitEmbedder__dropout.p = 0.0
    grads = native_grads(m, torch.from_numpy(g["chars"]).to(DEV), torch.from_numpy(g["grad_out"]).to(DEV))
    for gn, key in zip(grads, ("conv_l1.weight", "conv_l1.bias", "conv_l2.weight", "conv_l2.bias", "conv_l3.weight")):
        ref = torch.from_numpy(g["grad::" + R.PRE + key]).to(DEV).double()
        assert float((gn.double() - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max()))


def test_status_word_raises_on_the_next_call():
    m = module(101, 63, DEFAULT)
    chars = torch.randint(0, 101, (50, 15), device=DEV)
    bad = chars.clone()
    bad[3, 4] = 101
    with torch.no_grad():
        m(bad)
        torch.cuda.synchronize()
        with pytest.raises(IndexError):
            m(chars)
        m(chars)                   # the word was reset
        with torch.no_grad():
            for p in m._params():
                p.mul_(1e5)
        m(chars)
        torch.cuda.synchronize()
        with pytest.raises(FloatingPointError):
            m(chars)


def test_capture_and_no_host_synchronisation():
    m = module(101, 127, DEFAULT)
    chars = torch.randint(0, 101, (1000, 15), device=DEV)
    with torch.no_grad():
        eager = m(chars)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            m(chars)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(chars)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            captured = m(chars)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(captured, eager)


def test_memory_is_bounded():
    m = module(101, 127, DEFAULT)
    chars = torch.randint(0, 101, (80_000, 15), device=DEV)
    with torch.no_grad():
        m(chars)                   # prepared weights kept
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = m(chars)
        torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= out.numel() * 4 + (1 << 20)
    # backward: the chunked workspace does not grow with B
    peaks = []
    for B in (8192, 24576):
        mt, ch, go = make_grad_case(B, seed=4)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = mt(ch)
        torch.cuda.synchronize()
        mid = torch.cuda.memory_allocated()
        (out * go).sum().backward()
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - mid)
    assert peaks[1] <= peaks[0] * 1.25 + (8 << 20), peaks


def test_pickle_and_deepcopy_of_a_used_module():
    m = module(101, 63, DEFAULT)
    chars = torch.randint(0, 101, (40, 15), device=DEV)
    with torch.no_grad():
        ref = m(chars)
        for other in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
            assert other._status is not m._status
            assert torch.equal(other(chars), ref)


def test_training_steps_match_library_restatement():
    """Two SGD steps of a VarMisuse-shaped model -- char embedder (D = 63) -> cat(is_candidate) -> two native MlpMessagePassingLayers
    at H = 64 over a random two-type graph -- against the same model with the char embedder restated on library ops (true fp32).  The
    layers aggregate with "sum": a "max" winner within rounding of the runner-up may legitimately differ between the two embedders."""
    from ptgnn_b200 import MlpMessagePassingLayer

    torch.manual_seed(21)
    N_, H = 2000, 64
    gen = torch.Generator().manual_seed(22)
    adj = [(torch.randint(0, N_, (6000,), generator=gen).to(DEV), torch.randint(0, N_, (6000,), generator=gen).to(DEV)) for _ in range(2)]
    emb = CharUnitEmbedder(101, H - 1, DEFAULT, 0.0).to(DEV)
    layers = torch.nn.ModuleList([MlpMessagePassingLayer(H, H, H, 2, "sum") for _ in range(2)]).to(DEV).train()
    emb_ref, layers_ref = copy.deepcopy(emb), copy.deepcopy(layers)
    chars = torch.randint(0, 101, (N_, 15), device=DEV, generator=torch.Generator(device=DEV).manual_seed(23))
    cand = (torch.rand(N_, 1, device=DEV, generator=torch.Generator(device=DEV).manual_seed(24)) < 0.3).float()
    target = torch.randn(N_, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(25))

    def step(e, ls, native):
        ps = list(e.parameters()) + list(ls.parameters())
        for p in ps:
            p.grad = None
        h = torch.cat([e(chars) if native else R.forward(chars, *e._params(), dtype=torch.float32), cand], dim=-1)
        for layer in ls:
            h = layer(h, adj)
        loss = ((h - target) ** 2).mean()
        loss.backward()
        with torch.no_grad():
            for p in ps:
                p -= 0.1 * p.grad
        return float(loss.detach())

    for _ in range(2):
        ln, lr = step(emb, layers, True), step(emb_ref, layers_ref, False)
        assert abs(ln - lr) <= 1e-4 * max(1.0, abs(lr))
    for a, b in zip(list(emb.parameters()) + list(layers.parameters()), list(emb_ref.parameters()) + list(layers_ref.parameters())):
        assert float((a - b).abs().max()) <= 1e-4 * max(1.0, float(b.abs().max()))
