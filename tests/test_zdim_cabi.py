"""CPU-side checks of latent sizes other than multiples of 64: any z_dim that is a multiple of 4 in [4, 1024] is accepted
by the ConvVAE and MlpVAE layout / workspace entry points with the reference's variable shapes, and everything else is
rejected with an error that names z_dim.  No compute entry point is called here."""
import ctypes as C

import numpy as np
import pytest
from harness import lib, library_state  # noqa: F401

Z_GOOD = (4, 32, 100, 1024)
Z_BAD = (0, 2, 65, 1028)


def _vae_shapes(lib, ct, z):
    n = lib.cpb_vae_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
    assert lib.cpb_vae_layout(ct, z, offs, sizes, shapes, C.byref(total)) == 0, lib.cpb_last_error()
    names = [lib.cpb_vae_tensor_name(i).decode() for i in range(n)]
    return names, [tuple(s for s in shapes[4 * i:4 * i + 4] if s > 0) for i in range(n)], list(offs), list(sizes), total.value


def _mlp_config(z, batch=8):
    from carla_ppo_b200 import _lib
    base = _lib.VaeConfig(batch, 3, z, _lib.LOSS_BCE, _lib.FRAME_F32, _lib.FRAME_F32, 1 / 255.0, 1.0, 0.0, 1.0)
    return _lib.MlpVaeConfig(base, 512, 256, 256, 512)


@pytest.mark.parametrize("z", Z_GOOD)
@pytest.mark.parametrize("ct", [3, 1])
def test_vae_layout_matches_reference_variables_at_any_multiple_of_4(lib, z, ct):
    from oracle.vae_oracle import param_shapes
    names, shapes, offs, sizes, total = _vae_shapes(lib, ct, z)
    ref = param_shapes(target_channels=ct, z_dim=z)
    assert names == list(ref.keys())
    assert shapes == [ref[k] for k in names]
    assert sizes == [int(np.prod(ref[k])) for k in names]
    spans = sorted((o, o + s) for o, s in zip(offs, sizes))
    assert all(o % 64 == 0 for o in offs) and all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    assert spans[-1][1] <= total and total % 64 == 0


@pytest.mark.parametrize("z", Z_GOOD)
def test_mlp_layout_matches_reference_variables_at_any_multiple_of_4(lib, z):
    from oracle.vae_oracle import mlp_param_shapes
    cfg = _mlp_config(z)
    n = lib.cpb_mlpvae_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
    assert lib.cpb_mlpvae_layout(C.byref(cfg), offs, sizes, shapes, C.byref(total)) == 0, lib.cpb_last_error()
    ref = mlp_param_shapes(z_dim=z)
    names = [lib.cpb_mlpvae_tensor_name(i).decode() for i in range(n)]
    assert sorted(names) == sorted(ref.keys())
    for i, name in enumerate(names):
        assert tuple(s for s in shapes[4 * i:4 * i + 4] if s > 0) == ref[name], name
        assert sizes[i] == int(np.prod(ref[name]))


@pytest.mark.parametrize("z", Z_GOOD)
def test_workspace_sizes_are_positive_and_grow_with_the_mode(lib, z):
    for batch in (1, 32):
        enc, fwd, trn = (lib.cpb_vae_workspace_bytes(batch, 3, z, m) for m in range(3))
        assert 0 < enc < fwd < trn, (z, batch, enc, fwd, trn)
        cfg = _mlp_config(z, batch)
        enc, fwd, trn = (lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), m) for m in range(3))
        assert 0 < enc < fwd < trn, (z, batch, enc, fwd, trn)


def test_latent_padding_costs_no_more_than_the_next_multiple_of_64(lib):
    """The library pads the latent to 64 * ceil(z / 64) columns inside the workspace; a z below that multiple needs at
    most the padded size's workspace plus the zero-padded weight copies."""
    for z, zp in ((4, 64), (32, 64), (100, 128), (1020, 1024)):
        for mode in range(3):
            a = lib.cpb_vae_workspace_bytes(32, 3, z, mode)
            b = lib.cpb_vae_workspace_bytes(32, 3, zp, mode)
            copies = 4 * (3 * 6144 * zp + 2 * zp) + 3 * 256
            assert b <= a <= b + copies, (z, mode, a, b)


@pytest.mark.parametrize("z", Z_BAD)
def test_other_latent_sizes_are_rejected_naming_z_dim(lib, z):
    total = C.c_int64()
    assert lib.cpb_vae_layout(3, z, None, None, None, C.byref(total)) == -1
    assert b"z_dim" in lib.cpb_last_error()
    assert lib.cpb_vae_workspace_bytes(32, 3, z, 0) < 0
    assert b"z_dim" in lib.cpb_last_error()
    cfg = _mlp_config(z)
    assert lib.cpb_mlpvae_layout(C.byref(cfg), None, None, None, C.byref(total)) == -1
    assert b"z_dim" in lib.cpb_last_error()
    assert lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), 0) < 0


def test_train_vae_cli_names_the_model_directory_after_any_z_dim():
    from carla_ppo_b200.vae import train_vae
    args = train_vae.build_parser().parse_args(["--z_dim", "32"])
    assert args.z_dim == 32
    assert "_zdim32_" in train_vae.default_model_name(args)
