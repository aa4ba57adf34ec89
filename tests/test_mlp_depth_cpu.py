"""CPU-side checks of the MlpVAE at any depth (1 to 8 hidden layers per side): the spec layout follows the reference's
tf.layers names and creation order, the two-per-side model is the same through the spec entry points as through the
legacy ones, malformed specs are refused before anything launches, and the any-depth oracle (tests/mlp_depth_oracle.py)
matches torch autograd and, at two layers per side, oracle.vae_oracle and the TF32 restatement bit for bit.  No compute
entry point runs a kernel here."""
import ctypes as C

import numpy as np
import pytest

import mlp_depth_oracle as mdo
import mlp_tf32_oracle
from helpers import rel_l2
from harness import lib, library_state, math_mode  # noqa: F401

DEFAULT = ((512, 256), (256, 512))
SHAPES = {"1x1": ((512,), (512,)), "3x2": ((1024, 512, 256), (256, 512)),
          "8x8": ((256, 224, 192, 160, 128, 96, 64, 32), (32, 64, 96, 128, 160, 192, 224, 256))}


def _base(batch, ct=3, z=64):
    from carla_ppo_b200 import _lib
    return _lib.VaeConfig(batch, ct, z, _lib.LOSS_BCE, _lib.FRAME_F32, _lib.FRAME_F32, 1 / 255.0, 1.0, 0.0, 1.0)


def _spec(batch, enc, dec, ct=3, z=64):
    from carla_ppo_b200 import _lib
    return _lib.MlpVaeSpec.of(_base(batch, ct, z), enc, dec)


def _layout(lib, spec):
    n = lib.cpb_mlpvae_spec_num_tensors(C.byref(spec))
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
    assert lib.cpb_mlpvae_spec_layout(C.byref(spec), offs, sizes, shapes, C.byref(total)) == 0
    names = [lib.cpb_mlpvae_spec_tensor_name(C.byref(spec), i).decode() for i in range(n)]
    return names, list(offs), list(sizes), [tuple(s for s in shapes[4 * i:4 * i + 4] if s > 0) for i in range(n)], total.value


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("ct,z", [(3, 64), (1, 32)])
def test_spec_layout_follows_the_reference_names_and_creation_order(lib, shape, ct, z):
    enc, dec = SHAPES[shape]
    spec = _spec(1, enc, dec, ct, z)
    names, offs, sizes, shapes, total = _layout(lib, spec)
    ref = mdo.param_shapes(target_channels=ct, z_dim=z, encoder_sizes=enc, decoder_sizes=dec)
    assert len(names) == 2 * (len(enc) + len(dec) + 3)
    assert names == list(ref)                                   # tf.layers creation order
    assert names[0] == "encoder/dense/kernel" and names[-1] == "decoder/dense_%d/bias" % len(dec)
    assert shapes == list(ref.values())
    assert sizes == [int(np.prod(s)) for s in ref.values()]
    assert all(o % 64 == 0 for o in offs)
    spans = sorted((o, o + s) for o, s in zip(offs, sizes))
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= total and total % 64 == 0
    at = dict(zip(names, offs))
    step_k = -(-(enc[-1] * z) // 64) * 64
    assert at["logstd_sqare/kernel"] == at["mean/kernel"] + step_k          # the two head kernels adjacent
    assert at["mean/bias"] == at["logstd_sqare/kernel"] + step_k            # then the two head biases
    assert at["logstd_sqare/bias"] == at["mean/bias"] + -(-z // 64) * 64
    assert lib.cpb_mlpvae_spec_tensor_name(C.byref(spec), len(names)) is None


@pytest.mark.parametrize("z", [32, 64])
@pytest.mark.parametrize("ct", [3, 1])
def test_two_per_side_spec_is_the_legacy_model(lib, z, ct):
    """Layout, names, workspace bytes and buffer offsets of the default shape are the same through both sets of entry
    points, in every math mode and workspace mode."""
    from carla_ppo_b200 import _lib
    (e1, e2), (d1, d2) = DEFAULT
    n = lib.cpb_mlpvae_num_tensors()
    assert n == 14 and lib.cpb_mlpvae_spec_num_tensors(C.byref(_spec(1, *DEFAULT, ct, z))) == 14
    for batch in (8, 512):
        spec = _spec(batch, *DEFAULT, ct, z)
        cfg = _lib.MlpVaeConfig(_base(batch, ct, z), e1, e2, d1, d2)
        names, offs, sizes, shapes, total = _layout(lib, spec)
        lo = (C.c_int64 * n)(); ls = (C.c_int64 * n)(); lsh = (C.c_int32 * (4 * n))(); lt = C.c_int64()
        assert lib.cpb_mlpvae_layout(C.byref(cfg), lo, ls, lsh, C.byref(lt)) == 0
        assert names == [lib.cpb_mlpvae_tensor_name(i).decode() for i in range(n)]
        assert offs == list(lo) and sizes == list(ls) and total == lt.value
        assert shapes == [tuple(s for s in lsh[4 * i:4 * i + 4] if s > 0) for i in range(n)]
        for mode in (_lib.MATH_SIMT, _lib.MATH_3XTF32, _lib.MATH_TF32):
            with math_mode(lib, mode):
                for ws in range(3):
                    a = lib.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), ws)
                    assert a > 0 and a == lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), ws), (mode, ws)
                    so = (C.c_int64 * 10)(); lo2 = (C.c_int64 * 10)()
                    assert lib.cpb_debug_mlpvae_spec_buffer_offsets(C.byref(spec), ws, so, 10) == 10
                    assert lib.cpb_debug_mlpvae_buffer_offsets(C.byref(cfg), ws, lo2, 10) == 10
                    assert list(so) == list(lo2)


def test_buffer_offsets_name_every_hidden_layer(lib):
    from carla_ppo_b200 import _lib
    enc, dec = SHAPES["3x2"]
    spec = _spec(16, enc, dec)
    n = len(enc) + len(dec) + 6
    offs = (C.c_int64 * n)()
    assert lib.cpb_debug_mlpvae_spec_buffer_offsets(C.byref(spec), _lib.WS_TRAIN, offs, n) == n
    x, h0, h1, h2, heads, z, g0, g1, logits, ga, gb = list(offs)
    assert x == 0 and h0 == 16 * 38400 * 4 and h1 == h0 + 16 * 1024 * 4 and h2 == h1 + 16 * 512 * 4 and heads == h2 + 16 * 256 * 4
    assert heads < z < g0 < g1 < logits < ga < gb
    assert g1 == g0 + 16 * 256 * 4 and logits == g1 + 16 * 512 * 4
    enc_only = (C.c_int64 * n)()
    assert lib.cpb_debug_mlpvae_spec_buffer_offsets(C.byref(spec), _lib.WS_ENCODE, enc_only, n) == n
    assert list(enc_only)[5:] == [-1] * 6


def _bad_specs():
    from carla_ppo_b200 import _lib
    empty = _lib.MlpVaeSpec.of(_base(4), (512,), (512,))
    empty.num_encoder = 0
    empty_dec = _lib.MlpVaeSpec.of(_base(4), (512,), (512,))
    empty_dec.num_decoder = 0
    nine = _lib.MlpVaeSpec.of(_base(4), (64,) * 8, (64,))
    nine.num_encoder = 9
    return {"empty encoder": empty, "empty decoder": empty_dec, "nine layers": nine,
            "width 100": _lib.MlpVaeSpec.of(_base(4), (512, 100), (256,))}


def test_malformed_specs_are_refused_before_anything_launches(lib):
    from carla_ppo_b200 import _lib
    lib.cpb_reset_launch_count()
    fake = C.c_void_p(256)          # never dereferenced: the spec is checked first
    for what, spec in _bad_specs().items():
        assert lib.cpb_mlpvae_spec_num_tensors(C.byref(spec)) == -1, what
        msg = lib.cpb_last_error()
        assert (b"hidden layers per side" in msg) if what != "width 100" else (b"multiples of 32" in msg and b"100" in msg), (what, msg)
        assert lib.cpb_mlpvae_spec_tensor_name(C.byref(spec), 0) is None
        assert lib.cpb_mlpvae_spec_layout(C.byref(spec), None, None, None, None) == -1
        assert lib.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), _lib.WS_TRAIN) < 0
        assert lib.cpb_debug_mlpvae_spec_buffer_offsets(C.byref(spec), 2, (C.c_int64 * 32)(), 32) == -1
        assert lib.cpb_mlpvae_spec_loss_grad(C.byref(spec), fake, fake, fake, fake, fake, fake, None, fake, 1 << 40, None) == -1
        assert lib.cpb_mlpvae_spec_encode(C.byref(spec), fake, fake, fake, None, None, fake, 1 << 40, None) == -1
        ppo = _lib.PpoConfig(); ppo.state_dim, ppo.num_actions, ppo.hidden1, ppo.hidden2 = 67, 2, 500, 300
        assert lib.cpb_mlpvae_encode_predict(C.byref(spec), fake, fake, fake, 3, C.byref(ppo), fake, None, fake, fake, fake,
                                             fake, None, fake, 1 << 40, fake, 1 << 40, None) == -1
    assert lib.cpb_launch_count() == 0


def test_mlp_vae_class_takes_any_depth_and_refuses_the_rest(tmp_path):
    from carla_ppo_b200.vae.models import MlpVAE
    vae = MlpVAE((80, 160, 3), z_dim=64, encoder_sizes=[1024, 512, 256], decoder_sizes=[256, 512],
                 model_dir=str(tmp_path / "a"))
    assert vae.encoder_sizes == (1024, 512, 256) and vae.encoded_shape == (256,)
    spec = vae._config(4)
    assert spec.num_encoder == 3 and list(spec.encoder_sizes)[:3] == [1024, 512, 256] and spec.num_decoder == 2
    with pytest.raises(ValueError):
        vae._mlp_config(4)                      # the legacy config describes two layers per side only
    two = MlpVAE((80, 160, 3), z_dim=64, model_dir=str(tmp_path / "b"))
    cfg = two._mlp_config(4)
    assert (cfg.enc1, cfg.enc2, cfg.dec1, cfg.dec2) == (512, 256, 256, 512)
    for enc, dec in (((), (512,)), ((512,), ()), ((64,) * 9, (64,)), ((512, 100), (256,)), ((16,), (32,)), ((8224,), (32,))):
        with pytest.raises(ValueError):
            MlpVAE((80, 160, 3), z_dim=64, encoder_sizes=enc, decoder_sizes=dec, model_dir=str(tmp_path / "c"))


def _inputs(n, z, ct, seed=0):
    rs = np.random.RandomState(seed)
    x = rs.rand(n, 80, 160, 3).astype(np.float32)
    y = x if ct == 3 else rs.rand(n, 80, 160, 1).astype(np.float32)
    return x, y, rs.randn(n, z)


@pytest.mark.parametrize("enc,dec", [((64,), (32,)), ((96, 64, 32), (32, 64))])
def test_any_depth_oracle_backward_matches_autograd(enc, dec):
    p = mdo.glorot_init(3, target_channels=1, z_dim=32, encoder_sizes=enc, decoder_sizes=dec)
    x, y, eps = _inputs(3, 32, 1)
    for loss, beta, tol in (("mse", 1.0, 0.0), ("bce", 2.0, 0.0), ("bce_v2", 1.0, 0.3)):
        a = mdo.loss_and_grads(p, x, y, eps, loss, beta, tol)
        b = mdo.torch_loss_and_grads(p, x, y, eps, loss, beta, tol)
        assert abs(a["recon"] - b["recon"]) < 1e-9 * abs(b["recon"]) and abs(a["kl"] - b["kl"]) < 1e-9 * max(abs(b["kl"]), 1)
        assert rel_l2(a["mean"], b["mean"]) < 1e-12 and rel_l2(a["logits"], b["logits"]) < 1e-12
        assert sorted(a["grads"]) == sorted(p)
        for k in a["grads"]:
            assert rel_l2(a["grads"][k], b["grads"][k]) < 1e-10, (loss, k)


@pytest.mark.parametrize("ct,z,enc,dec", [(1, 32, (96, 64), (160, 64)), (3, 64, (64, 32), (32, 64))])
def test_at_two_per_side_the_any_depth_oracle_is_the_oracle_bit_for_bit(ct, z, enc, dec):
    """Shapes, initial weights, loss, gradients and an Adam step equal oracle.vae_oracle's; with the TF32 hook the
    result equals the TF32 restatement tests/mlp_tf32_oracle.py."""
    from oracle import vae_oracle as vo
    kw = dict(target_channels=ct, z_dim=z, encoder_sizes=enc, decoder_sizes=dec)
    assert mdo.param_shapes(**kw) == vo.mlp_param_shapes(**kw)
    w = mdo.glorot_init(2, **kw)
    ow = vo.mlp_glorot_init(2, **kw)
    assert list(w) == list(ow) and all(np.array_equal(w[k], ow[k]) for k in w)
    x, y, eps = _inputs(3, z, ct, 5)
    got = mdo.loss_and_grads(w, x, y, eps, "bce_v2", beta=2.0, kl_tolerance=0.1)
    ref = vo.mlp_loss_and_grads(w, x, y, eps, "bce_v2", beta=2.0, kl_tolerance=0.1)
    for k in ("mean", "logvar", "z", "logits"):
        assert np.array_equal(got[k], ref[k]), k
    assert got["recon"] == ref["recon"] and got["kl"] == ref["kl"]
    assert sorted(got["grads"]) == sorted(ref["grads"])
    assert all(np.array_equal(got["grads"][k], ref["grads"][k]) for k in ref["grads"])
    pa = {k: v.astype(np.float64) for k, v in w.items()}
    pb = {k: v.astype(np.float64) for k, v in w.items()}
    sa, sb = vo.adam_init_state(pa), vo.adam_init_state(pb)
    assert mdo.train_step(pa, sa, x, y, eps, loss_type="mse") == vo.mlp_train_step(pb, sb, x, y, eps, loss_type="mse")
    assert all(np.array_equal(pa[k], pb[k]) for k in pa)
    for hook in (None, mlp_tf32_oracle.round_tf32):
        got = mdo.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, tc_round=hook)
        ref = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, tc_round=hook or (lambda a: a))
        for k in ("mean", "logvar", "z", "logits"):
            assert np.array_equal(got[k], ref[k]), (hook, k)
        assert got["recon"] == ref["recon"] and got["kl"] == ref["kl"]
        assert sorted(got["grads"]) == sorted(ref["grads"])
        assert all(np.array_equal(got["grads"][k], ref["grads"][k]) for k in ref["grads"]), hook
    # with the run's own ReLU pattern the masked form is the same function
    own = mdo.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1)
    ri = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, tc_round=lambda a: a)["relu_inputs"]
    masks = {"h0": ri["h1"] > 0, "h1": ri["h2"] > 0, "g0": ri["g1"] > 0, "g1": ri["g2"] > 0}
    again = mdo.loss_and_grads(w, x, y, eps, "bce", kl_tolerance=0.1, relu_masks=masks)
    assert all(np.allclose(again["grads"][k], own["grads"][k], rtol=1e-12, atol=0) for k in own["grads"])


def test_rounding_hook_touches_exactly_the_five_frame_wide_products():
    """At three encoder and two decoder layers: a hook that records its calls sees the two operands of each of the five
    products, and every such pair reduces over or produces a frame (38 400 or 12 800 long on some axis)."""
    w = mdo.glorot_init(4, target_channels=1, z_dim=32, encoder_sizes=(96, 64, 32), decoder_sizes=(32, 64))
    x, y, eps = _inputs(2, 32, 1, 7)
    seen = []

    def hook(a):
        seen.append(a.shape)
        return a
    out = mdo.loss_and_grads(w, x, y, eps, "mse", tc_round=hook)
    assert len(seen) == 10
    for a, b in zip(seen[0::2], seen[1::2]):
        assert {38400, 12800} & set(a + b), (a, b)
    plain = mdo.loss_and_grads(w, x, y, eps, "mse")
    assert all(np.array_equal(out["grads"][k], plain["grads"][k]) for k in plain["grads"])
