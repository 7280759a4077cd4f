"""CPU checks of the native ``LinearFeatureEmbedder`` (DESIGN.md §3.15): constructor, ``state_dict`` keys and seeded parameters against
the reference class, the size query, the refusals (raised before any kernel runs) and the ``overlay.install(native_feature_embedder=True)``
binding."""
import inspect
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from oracle.refimport import import_reference, reference_available

import ptgnn_b200
from ptgnn_b200 import _native as N
from ptgnn_b200 import embeddings as EMB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULE = "ptgnn.neuralmodels.embeddings.linearmapembedding"
KEY = "_LinearFeatureEmbedder__linear_map.weight"
needs_reference = pytest.mark.skipif(not reference_available(), reason="the reference tree is not present")


def test_constructor_signature_and_keys():
    cls = ptgnn_b200.LinearFeatureEmbedder
    params = inspect.signature(cls.__init__).parameters
    assert list(params) == ["self", "input_element_size", "output_embedding_size", "activation"]
    assert params["activation"].default is None
    assert list(inspect.signature(cls.forward).parameters) == ["self", "features"]
    m = cls(50, 64, nn.ReLU())
    assert list(m.state_dict()) == [KEY] and tuple(m.state_dict()[KEY].shape) == (64, 50)


@needs_reference
def test_seeded_parameters_and_state_dicts_match_the_reference():
    import warnings

    import_reference()
    ref = __import__(MODULE, fromlist=["x"])
    for F, D, act in ((50, 64, None), (1, 8, nn.Tanh()), (121, 256, nn.GELU())):
        torch.manual_seed(11)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", FutureWarning)      # the reference calls the deprecated nn.init.xavier_uniform
            r = ref.LinearFeatureEmbedder(F, D, act)
        torch.manual_seed(11)
        n = ptgnn_b200.LinearFeatureEmbedder(F, D, act)
        sig = lambda cls: [(q.name, q.default) for q in inspect.signature(cls.__init__).parameters.values()]
        assert sig(type(r)) == sig(type(n))
        assert list(r.state_dict()) == list(n.state_dict())
        assert all(torch.equal(a, b) for a, b in zip(r.state_dict().values(), n.state_dict().values()))
        n.load_state_dict(r.state_dict(), strict=True)
        r.load_state_dict(n.state_dict(), strict=True)


# (bf16, in_dim, out_dim) -> bytes of the prepared weights; 0 marks an unsupported shape
_PREPARED = {(0, 50, 64): 16384, (1, 50, 64): 8192, (0, 121, 256): 131072, (0, 512, 256): 524288, (1, 512, 256): 262144,
             (0, 1, 8): 4096, (0, 50, 12): 0, (0, 0, 64): 0, (0, 513, 64): 0, (0, 50, 264): 0}


def test_supported_shapes_and_prepared_sizes_are_pinned():
    lib = N.lib()
    for (bf16, F, D), want in _PREPARED.items():
        assert lib.ptgnn_b200_feature_embed_workspace_bytes(bf16, F, D) == want, (bf16, F, D)
        assert bool(lib.ptgnn_b200_feature_embed_supported(F, D)) == (want > 0), (F, D)


def test_refusals_before_any_kernel(monkeypatch):
    launches = N.launch_count()
    x = torch.zeros(3, 50)
    with pytest.raises(NotImplementedError, match="multiple of 8"):
        ptgnn_b200.LinearFeatureEmbedder(50, 12)(x)
    with pytest.raises(NotImplementedError):
        ptgnn_b200.LinearFeatureEmbedder(600, 64)(torch.zeros(3, 600))
    with pytest.raises(NotImplementedError, match="no native kernel"):
        ptgnn_b200.LinearFeatureEmbedder(50, 64, nn.Sigmoid())(x)
    with pytest.raises(NotImplementedError, match="no native kernel"):
        ptgnn_b200.LinearFeatureEmbedder(50, 64, nn.GELU(approximate="tanh"))(x)
    monkeypatch.setattr(EMB, "_bf16_autocast", lambda device: True)
    with pytest.raises(NotImplementedError, match="gradients with a bf16 output"):
        ptgnn_b200.LinearFeatureEmbedder(50, 64, nn.ReLU())(x)
    assert N.launch_count() == launches


def test_cpu_tensors_raise():
    with torch.no_grad(), pytest.raises(N.NativeLibraryError):
        ptgnn_b200.LinearFeatureEmbedder(50, 64)(torch.zeros(3, 50))


def test_scratch_is_not_pickled_or_deep_copied():
    import copy
    import pickle

    m = ptgnn_b200.LinearFeatureEmbedder(50, 64, nn.Tanh())
    m._status, m._transformed = torch.zeros(1, dtype=torch.int32), ("key", torch.zeros(8, dtype=torch.uint8))
    for restored in (pickle.loads(pickle.dumps(m)), copy.deepcopy(m)):
        assert restored._status is None and restored._transformed is None
        assert torch.equal(restored.state_dict()[KEY], m.state_dict()[KEY])


@needs_reference
def test_overlay_binds_the_native_feature_embedder_only_when_asked():
    code = (
        "import sys, warnings; sys.path.insert(0, %r)\n"
        "warnings.simplefilter('ignore', FutureWarning)\n"
        "from oracle.refimport import import_reference\nimport_reference()\n"
        "import ptgnn_b200 as P, ptgnn_b200.overlay as ov, importlib\n"
        "MOD = %r\n"
        "mod = importlib.import_module(MOD)\nref = mod.LinearFeatureEmbedder\n"
        "def build():\n"
        "    model = mod.FeatureRepresentationModel(embedding_size=64)\n"
        "    model._FeatureRepresentationModel__num_input_features = 50\n"
        "    return model.build_neural_module()\n"
        "r = ov.install(force_torch_scatter=True)\n"
        "assert r['feature_embedder'] is False and mod.LinearFeatureEmbedder is ref and type(build()) is ref\n"
        "ov.uninstall()\n"
        "holder = type(sys)('holder'); holder.__name__ = 'ptgnn.holder'; holder.LFE = ref; sys.modules['ptgnn.holder'] = holder\n"
        "r = ov.install(force_torch_scatter=True, native_feature_embedder=True)\n"
        "assert r['feature_embedder'] is True and mod.LinearFeatureEmbedder is P.LinearFeatureEmbedder\n"
        "assert holder.LFE is P.LinearFeatureEmbedder, 'a reference module imported before install is re-bound'\n"
        "m = build()\nassert type(m) is P.LinearFeatureEmbedder and list(m.state_dict()) == [%r]\n"
        "ov.uninstall()\n"
        "assert mod.LinearFeatureEmbedder is ref and holder.LFE is ref and type(build()) is ref\nprint('FEATURE-OVERLAY-OK')\n"
        % (ROOT, MODULE, KEY))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and "FEATURE-OVERLAY-OK" in r.stdout, r.stdout + r.stderr[-3000:]
