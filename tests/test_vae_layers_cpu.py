"""Pins the torch formulation the per-layer GPU tests use as their reference (tests/vae_layer_ref.py) to the float64
oracle's primitives, on the CPU: the three contractions at both kernel sizes, the channel counts of the edge layers
(3 and 1) and of the interior ones, odd output sizes and B = 1 and 3; the z_pad handling of the dense layers; and the
TF32 rounding against tests/tf32_oracle.py."""
import numpy as np
import pytest
import torch

import vae_layer_ref as R
from oracle import vae_oracle as vo
from tf32_oracle import round_tf32

TOL = 1e-12


def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


# (k, Cb, Cs, Hs, Ws): the big image is (2 (Hs - 1) + k) x (2 (Ws - 1) + k) plus `extra` rows / columns the kernel
# never reaches (conv4's 8 x 18 input gives 3 x 8 and leaves its last row and column out, as 80 x 160 -> 39 x 79 does)
SHAPES = [(4, 3, 32, 5, 7), (4, 1, 32, 3, 9), (5, 32, 64, 4, 5), (4, 32, 64, 3, 3), (5, 3, 8, 1, 1), (4, 64, 16, 1, 2)]


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("k,cb,cs,hs,ws", SHAPES)
def test_torch_contractions_match_the_oracle(k, cb, cs, hs, ws, extra, batch):
    rs = np.random.RandomState(k * 1000 + cb * 10 + cs + extra + batch)
    hb, wb = 2 * (hs - 1) + k + extra, 2 * (ws - 1) + k + extra
    big = rs.randn(batch, hb, wb, cb)
    small = rs.randn(batch, hs, ws, cs)
    w = rs.randn(k, k, cb, cs)
    t = lambda a: torch.from_numpy(a)
    got = R.gather(t(big), t(w)).numpy()
    assert got.shape == (batch, hs, ws, cs)
    assert _rel(got, vo.conv_gather(big, w)) < TOL
    got = R.scatter(t(small), t(w), (hb, wb)).numpy()
    assert got.shape == big.shape
    assert _rel(got, vo.conv_scatter(small, w, out_hw=(hb, wb))) < TOL
    got = R.wgrad(t(big), t(small), k).numpy()
    assert _rel(got, vo.conv_wgrad(big, small, k)) < TOL
    # a non-contiguous view (the device's 4-channel padded frames are sliced to their Ct channels)
    padded = np.concatenate([big, rs.randn(batch, hb, wb, 1)], axis=3)
    assert _rel(R.gather(t(padded)[..., :cb], t(w)).numpy(), vo.conv_gather(big, w)) < TOL
    assert _rel(R.wgrad(t(padded)[..., :cb], t(small), k).numpy(), vo.conv_wgrad(big, small, k)) < TOL


@pytest.mark.parametrize("z", [64, 100, 4])
def test_dense_layers_drop_the_padded_latent_columns(z):
    """The library keeps the latent rows (z, gz, gheads) at a pitch of z_pad = 64 ceil(z / 64) columns.  The reference
    reads the first z columns of such a buffer, whatever the padding holds, and gives the oracle's products on the
    unpadded [B, z] rows: the latent side of dense1 and of the heads' data gradient."""
    rs = np.random.RandomState(z)
    zp = 64 * ((z + 63) // 64)
    b, feat = 3, 96
    wm, wl, wd = rs.randn(feat, z), rs.randn(feat, z), rs.randn(z, feat)
    lat, gm, gl = rs.randn(b, z), rs.randn(b, z), rs.randn(b, z)
    lat_p = np.full((b, zp), np.nan); lat_p[:, :z] = lat
    gh_p = np.full((2, b, zp), np.nan); gh_p[0, :, :z] = gm; gh_p[1, :, :z] = gl
    t = torch.from_numpy
    assert _rel(R.dense1_fwd(t(lat_p), t(wd)).numpy(), lat @ wd) < TOL
    # vae_oracle.loss_and_grads: gflat = gmean @ mean/kernel^T + glogvar @ logstd_sqare/kernel^T
    assert _rel(R.heads_dgrad(t(gh_p), t(wm), t(wl)).numpy(), gm @ wm.T + gl @ wl.T) < TOL


STOPS = ["deconv4.dgrad", "deconv3.dgrad", "deconv2.dgrad", "deconv1.dgrad", "dense1.dgrad", "heads.dgrad",
         "conv4.dgrad", "conv3.dgrad"]


def test_backward_stop_hook_accepts_exactly_the_layer_groups():
    import ctypes as C
    import os
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = _lib.load()
    try:
        for g in STOPS:
            assert lib.cpb_debug_vae_backward_stop(g.encode()) == 0
        for bad in (b"conv2.dgrad", b"conv1.wgrad", b"deconv4", b"", b"heads.dgrad "):
            assert lib.cpb_debug_vae_backward_stop(bad) == -1
            assert b"unknown layer group" in lib.cpb_last_error()
    finally:
        assert lib.cpb_debug_vae_backward_stop(None) == 0
    # gz and gheads follow kl_rows in the buffer table; only the training workspace has them
    offs = (C.c_int64 * 20)()
    for mode, present in ((_lib.WS_FORWARD, False), (_lib.WS_TRAIN, True)):
        assert lib.cpb_debug_vae_buffer_offsets(33, 3, 100, mode, offs, 20) == 18
        assert (offs[16] >= 0) == present and (offs[17] >= 0) == present
    assert offs[17] - offs[16] == 4 * 33 * 128          # gz is [B, z_pad] with z_pad = 128 at z = 100
    # a caller sized for the 16-entry table gets those 16 entries, and the count it asked for, and nothing past them
    short = (C.c_int64 * 17)(*([-7] * 17))
    assert lib.cpb_debug_vae_buffer_offsets(33, 3, 100, _lib.WS_TRAIN, short, 16) == 16
    assert list(short[:16]) == list(offs[:16]) and short[16] == -7
    assert lib.cpb_debug_vae_buffer_offsets(33, 3, 100, _lib.WS_TRAIN, short, 0) == 0


def test_round_tf32_matches_the_tf32_restatement():
    rs = np.random.RandomState(0)
    a = np.concatenate([rs.randn(4096).astype(np.float32) * np.float32(10.0) ** rs.randint(-20, 20, 4096),
                        np.float32([0.0, -0.0, 1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, -1.0 - 2 ** -11, 3.4e38, -3.4e38, 1e-40])])
    got = R.round_tf32(torch.from_numpy(a)).numpy()
    assert got.dtype == np.float32
    assert np.array_equal(got.astype(np.float64), round_tf32(a))
