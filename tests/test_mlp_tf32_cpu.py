"""CPU-side checks of math mode 2 on the MlpVAE: the TF32 restatement (tests/mlp_tf32_oracle.py) is the oracle when
nothing is rounded and rounds exactly the five frame-wide products; the workspace grows by exactly the TF32 weight
images and split partials in mode 2 and not at all in modes 0 and 1.  No compute entry point is called here."""
import ctypes as C

import numpy as np
import pytest

import mlp_tf32_oracle
from harness import lib, library_state, math_mode  # noqa: F401

IN, TBK, WAVE = 38400, 32, 132


def _cfg(batch, ct=3, z=64, sizes=(512, 256, 256, 512)):
    from carla_ppo_b200 import _lib
    base = _lib.VaeConfig(batch, ct, z, _lib.LOSS_BCE, _lib.FRAME_F32, _lib.FRAME_F32, 1 / 255.0, 1.0, 0.0, 1.0)
    return _lib.MlpVaeConfig(base, *sizes)


def test_restatement_is_the_oracle_with_five_products_rounded():
    from oracle import vae_oracle as vo
    w = vo.mlp_glorot_init(2, target_channels=1, z_dim=32, encoder_sizes=(96, 64), decoder_sizes=(160, 64))
    x = np.random.RandomState(0).rand(3, 80, 160, 3).astype(np.float32)
    y = np.random.RandomState(1).rand(3, 80, 160, 1).astype(np.float32)
    eps = np.random.RandomState(2).randn(3, 32).astype(np.float32)
    ref = vo.mlp_loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1)
    calls = {}
    same = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, tc_round=lambda a: a, calls=calls)
    assert calls == {"rounded": 5, "plain": 15}
    for k in ("mean", "logvar", "z", "logits"):
        assert np.array_equal(same[k], ref[k]), k
    assert same["recon"] == ref["recon"] and same["kl"] == ref["kl"]
    assert all(np.array_equal(same["grads"][k], ref["grads"][k]) for k in ref["grads"])
    # with the ReLU masks of the run itself, the masked form is the same function
    masks = {k: v > 0 for k, v in same["relu_inputs"].items()}
    again = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, tc_round=lambda a: a, relu_masks=masks)
    assert all(np.allclose(again["grads"][k], ref["grads"][k], rtol=1e-12, atol=0) for k in ref["grads"])
    t32 = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1)
    assert not np.array_equal(t32["mean"], ref["mean"])
    # the rounded-operand product is exactly what the restatement computes for encoder/dense
    h1 = np.maximum(mlp_tf32_oracle.round_tf32(x.reshape(3, -1)) @ mlp_tf32_oracle.round_tf32(w["encoder/dense/kernel"])
                    + w["encoder/dense/bias"], 0.0)
    assert np.array_equal(h1, t32["relu_inputs"]["h1"])


def _ksplit(K):
    return min(4, max(1, -(-(K // TBK) // 320)))


def _wg_splits(I, J, M):
    tiles = -(-I // 128) * (J // (64 if J % 64 == 0 else 32))
    return max(1, min(WAVE // tiles, (M + 1023) // 1024))


def _align(nbytes, a=256):
    return -(-nbytes // a) * a


def _mode2_extra(batch, ct, sizes, ws_mode):
    """Bytes mode 2 adds to a workspace, from the shapes: the TF32 weight images (2 x N x K floats each: the tensor-core
    operand layout interleaves a hi and a lo image) and one scratch for the split partials."""
    e1, _, _, d2 = sizes
    out = 12800 * ct
    images = 2 * e1 * IN
    scratch = _ksplit(IN) * batch * e1
    if ws_mode >= 1:
        images += 2 * out * d2
    if ws_mode >= 2:
        images += 2 * d2 * out
        scratch = max(scratch, _ksplit(out) * batch * d2, _wg_splits(IN, e1, batch) * IN * e1,
                      _wg_splits(out, d2, batch) * out * d2)
    return _align(4 * images) + _align(4 * scratch)


@pytest.mark.parametrize("batch,ct,z,sizes", [(8, 3, 64, (512, 256, 256, 512)), (512, 3, 64, (512, 256, 256, 512)),
                                              (4096, 3, 64, (512, 256, 256, 512)), (6, 1, 32, (96, 64, 160, 64)),
                                              (300, 1, 100, (32, 32, 32, 32))])
def test_workspace_grows_by_the_tf32_images_and_partials_in_mode_2_only(lib, batch, ct, z, sizes):
    from carla_ppo_b200 import _lib
    cfg = _cfg(batch, ct, z, sizes)
    size = {}
    for mode in (_lib.MATH_SIMT, _lib.MATH_3XTF32, _lib.MATH_TF32):
        with math_mode(lib, mode):
            size[mode] = [lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), ws) for ws in range(3)]
    assert size[_lib.MATH_SIMT] == size[_lib.MATH_3XTF32]
    for ws in range(3):
        assert size[_lib.MATH_TF32][ws] - size[_lib.MATH_3XTF32][ws] == _mode2_extra(batch, ct, sizes, ws), ws


def test_buffer_offsets_hook_names_the_mlp_buffers_and_ignores_the_math_mode(lib):
    from carla_ppo_b200 import _lib
    cfg = _cfg(16)
    got = {}
    for mode in (_lib.MATH_3XTF32, _lib.MATH_TF32):
        with math_mode(lib, mode):
            for ws in range(3):
                offs = (C.c_int64 * 10)()
                assert lib.cpb_debug_mlpvae_buffer_offsets(C.byref(cfg), ws, offs, 10) == 10
                got[mode, ws] = list(offs)
    for ws in range(3):
        assert got[_lib.MATH_3XTF32, ws] == got[_lib.MATH_TF32, ws]
    x, h1, h2, heads, z, g1, g2, logits, ga, gb = got[_lib.MATH_3XTF32, 2]
    assert x == 0 and h1 == 16 * IN * 4 and h2 == h1 + 16 * 512 * 4 and heads == h2 + 16 * 256 * 4
    assert min(z, g1, g2, logits, ga, gb) > heads
    assert got[_lib.MATH_3XTF32, 0][4:] == [-1] * 6 and got[_lib.MATH_3XTF32, 1][8:] == [-1, -1]
    bad = _cfg(16, sizes=(500, 256, 256, 512))
    assert lib.cpb_debug_mlpvae_buffer_offsets(C.byref(bad), 2, (C.c_int64 * 10)(), 10) == -1
    assert lib.cpb_debug_mlpvae_buffer_offsets(C.byref(cfg), 3, (C.c_int64 * 10)(), 10) == -1
