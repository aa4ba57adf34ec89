"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the header declares,
its layout tables agree with the reference's variable shapes, and bad arguments are rejected without a GPU.
No compute entry point is called here."""
import ctypes as C
import os
import re

import numpy as np
import pytest
from harness import lib, library_state  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    with open(os.path.join(ROOT, "include", "carla_ppo_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(cpb_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from carla_ppo_b200 import _lib
    declared = header_functions()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), "header declares %s but the library does not export it" % name
        assert name in _lib.PROTOTYPES, "%s has no ctypes prototype" % name
    assert sorted(_lib.PROTOTYPES) == declared


def test_vae_layout_matches_reference_variables(lib):
    from oracle.vae_oracle import param_shapes
    for ct in (3, 1):
        n = lib.cpb_vae_num_tensors()
        offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
        assert lib.cpb_vae_layout(ct, 64, offs, sizes, shapes, C.byref(total)) == 0
        ref = param_shapes(target_channels=ct)
        names = [lib.cpb_vae_tensor_name(i).decode() for i in range(n)]
        assert names == list(ref.keys())                        # TF creation order
        spans = []
        for i, name in enumerate(names):
            shape = tuple(s for s in shapes[4 * i:4 * i + 4] if s > 0)
            assert shape == ref[name], name
            assert sizes[i] == int(np.prod(ref[name]))
            assert offs[i] % 64 == 0
            spans.append((offs[i], offs[i] + sizes[i]))
        spans.sort()
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))   # no overlap
        assert spans[-1][1] <= total.value and total.value % 64 == 0
        assert sum(sizes) == (2584387 if ct == 3 else 2584387 - 2 * (16 * 32 + 1))
    assert lib.cpb_vae_tensor_name(99) is None


def test_ppo_layout_matches_reference_variables(lib):
    from carla_ppo_b200 import _lib
    from oracle.ppo_oracle import param_shapes, PPO_TENSORS
    cfg = _lib.PpoConfig(); cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = 67, 2, 500, 300
    n = lib.cpb_ppo_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (2 * n))(); total = C.c_int64()
    assert lib.cpb_ppo_layout(C.byref(cfg), offs, sizes, shapes, C.byref(total)) == 0
    names = [lib.cpb_ppo_tensor_name(i).decode() for i in range(n)]
    assert names == PPO_TENSORS
    ref = param_shapes()
    for i, name in enumerate(names):
        assert tuple(s for s in shapes[2 * i:2 * i + 2] if s > 0) == ref[name]
    assert sum(sizes) == 369505


def test_workspace_sizes_and_argument_errors(lib):
    enc = lib.cpb_vae_workspace_bytes(32, 3, 64, 0)
    fwd = lib.cpb_vae_workspace_bytes(32, 3, 64, 1)
    trn = lib.cpb_vae_workspace_bytes(32, 3, 64, 2)
    assert 0 < enc < fwd < trn
    assert lib.cpb_vae_workspace_bytes(4096, 3, 64, 2) < 20e9           # fits an 80 GB H100 several times over
    assert lib.cpb_vae_workspace_bytes(0, 3, 64, 2) < 0
    assert lib.cpb_vae_workspace_bytes(32, 2, 64, 2) < 0
    assert b"bad arguments" in lib.cpb_last_error()
    total = C.c_int64()
    assert lib.cpb_vae_layout(3, 65, None, None, None, C.byref(total)) == -1    # z_dim must be a multiple of 64
    assert b"z_dim" in lib.cpb_last_error()
    from carla_ppo_b200 import _lib
    with pytest.raises(_lib.CpbError):
        _lib.check(lib.cpb_vae_layout(5, 64, None, None, None, None), "cpb_vae_layout")
    assert b"sm_90a" in lib.cpb_build_info()


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under carla_ppo_b200/ may reference it."""
    pkg = os.path.join(ROOT, "carla_ppo_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".sh")):
                with open(os.path.join(dirpath, fn)) as f:
                    text = f.read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), os.path.join(dirpath, fn)
                assert "/root/reference" not in text, os.path.join(dirpath, fn)


def test_classes_fail_loudly_without_cuda(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from carla_ppo_b200._lib import CpbError
    from carla_ppo_b200.vae.models import ConvVAE, MlpVAE, bce_loss, bce_loss_v2, mse_loss
    vae = ConvVAE((80, 160, 3), z_dim=64, model_dir=str(tmp_path / "v"), models_dir="vae")
    assert vae.z_dim == 64 and vae.sample.shape[1] == 64 and vae.target_shape == (80, 160, 3)
    assert os.path.isdir(vae.checkpoint_dir) and os.path.isdir(vae.log_dir)
    with pytest.raises(CpbError):
        vae.init_session()                       # no CPU fallback
    with pytest.raises(CpbError):
        vae.encode(np.zeros((1, 80, 160, 3), np.float32))
    mlp = MlpVAE((80, 160, 3), z_dim=64, model_dir=str(tmp_path / "mlp"))     # reference vae/models.py:271-299
    assert mlp.encoder_sizes == (512, 256) and mlp.decoder_sizes == (256, 512)
    with pytest.raises(CpbError):
        mlp.init_session()                       # no CPU fallback either
    with pytest.raises(ValueError):
        ConvVAE((64, 64, 3), model_dir=str(tmp_path / "w"))
    x = np.array([0.3, -1.2]); y = np.array([1.0, 0.0])
    s = 1 / (1 + np.exp(-x))
    assert np.allclose(bce_loss(y, x, s), -(y * np.log(s) + (1 - y) * np.log(1 - s)))
    assert np.allclose(bce_loss_v2(y, x, s), bce_loss(y, x, s), atol=1e-8)
    assert np.allclose(mse_loss(y, x, s), (y - s) ** 2)
