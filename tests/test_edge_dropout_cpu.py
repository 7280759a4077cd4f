"""The per-edge dropout mask of GatedMessagePassingLayer (ptgnn_b200/csrc/edge_dropout.cuh), restated in numpy: Philox4x32-10 against
the Random123 known-answer vectors, keep fractions on fixed keys, p = 1, and the configurations that still refuse."""
import math

import numpy as np
import pytest
import torch

import edge_dropout_reference as R


@pytest.mark.parametrize("ctr, key, expected", [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0], [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
])
def test_philox_known_answers(ctr, key, expected):
    assert R.philox4x32_10(np.array([ctr], dtype=np.uint32), key)[0].tolist() == expected


@pytest.mark.parametrize("p", [0.01, 0.1, 0.5])
@pytest.mark.parametrize("key", [(0x12345678, 0x9ABCDEF0), (7, 0)])
def test_keep_fraction_within_six_sigma(p, key):
    E, K = 2048, 128
    n = E * K
    kept = int(R.keep_mask(key, E, K, p).sum())
    # binomial(n, 1 - p): a fixed key makes this deterministic, 6 sigma keeps it far from any edge
    assert abs(kept - n * (1 - p)) <= 6 * math.sqrt(n * p * (1 - p))


def test_p_one_drops_everything_and_p_zero_keeps_everything():
    assert not R.keep_mask((1, 2), 64, 64, 1.0).any()
    assert R.scale(1.0) == 0.0
    assert R.keep_mask((1, 2), 64, 64, 0.0).all()


def test_bits_layout():
    mask = R.keep_mask((3, 4), 5, 64, 0.3)
    bits = R.keep_bits(mask).view(np.uint32)
    for e in range(5):
        for k in range(64):
            assert bool((int(bits[e, k // 32]) >> (k % 32)) & 1) == bool(mask[e, k])


def test_unsupported_dropout_configurations_still_refuse():
    """bf16 states and node-range shards with training-mode dropout keep raising before any kernel runs."""
    from ptgnn_b200 import messagepassing as P

    adj = [(torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int64))]
    layer = P.GatedMessagePassingLayer(128, 128, 1, "sum", dropout_rate=0.1).train()
    with pytest.raises(NotImplementedError):
        layer(torch.zeros(4, 128, dtype=torch.bfloat16), adj)
    with pytest.raises(NotImplementedError):
        layer(torch.zeros(4, 128), adj, gather_states=torch.zeros(8, 128))
