"""Which MlpMessagePassingLayer configurations train with bf16 node states (no GPU needed): the supported ones get past the
refusal to the device checks, every other one raises NotImplementedError."""
import pytest
import torch

import ptgnn_b200 as P
from ptgnn_b200 import _native as N
from ptgnn_b200.messagepassing import _mlp_bf16_grad_supported

ADJ = [(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))]


def _bf16(H):
    return torch.zeros(4, H, dtype=torch.bfloat16, requires_grad=True)


@pytest.mark.parametrize("H,D", [(64, 128), (128, 128), (256, 128), (64, 64), (128, 64), (96, 128), (128, 256)])
@pytest.mark.parametrize("use_target", [True, False])
def test_supported_dims_reach_the_device_checks(H, D, use_target):
    assert _mlp_bf16_grad_supported(N.lib(), H, D, use_target)
    with pytest.raises(N.NativeLibraryError):      # CPU tensors: past the refusal, stopped where the states go to the device
        P.MlpMessagePassingLayer(H, H, D, 1, "max", use_target_state_as_message_input=use_target)(_bf16(H), ADJ)


@pytest.mark.parametrize("H,D", [(32, 32), (32, 128), (128, 48)])
def test_unsupported_dims_refuse(H, D):
    assert not _mlp_bf16_grad_supported(N.lib(), H, D, True)
    with pytest.raises(NotImplementedError):
        P.MlpMessagePassingLayer(H, H, D, 1, "sum")(_bf16(H), ADJ)


def test_other_configurations_refuse_with_bf16_gradients():
    for layer in (P.MlpMessagePassingLayer(128, 128, 128, 1, "sum", mlp_hidden_layers=1),
                  P.MlpMessagePassingLayer(128, 128, 128, 1, "sum", features_dimension=4),
                  P.MlpMessagePassingLayer(128, 128, 128, 1, P.PnaMessageAggregation())):
        with pytest.raises(NotImplementedError):
            layer(_bf16(128), ADJ)
    with pytest.raises(NotImplementedError):       # sharded
        P.MlpMessagePassingLayer(128, 128, 128, 1, "sum")(_bf16(128), ADJ, gather_states=torch.zeros(4, 128, dtype=torch.bfloat16))
