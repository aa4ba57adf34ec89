"""CPU-side checks of the ConvVAE at every frame size the reference builds (H and W multiples of 16 in [48, 512]): the
cpb_vae_spec_* layout against the oracle's variable shapes, the legacy 80x160 entry points against their spec twins,
refusals that happen before any memory is touched, the oracle's backward against torch autograd away from 80x160, and
the Python classes' constructor rule.  No compute entry point reaches the device here."""
import ctypes as C

import numpy as np
import pytest

from helpers import rel_l2
from harness import lib, library_state, math_mode  # noqa: F401

SIDES = list(range(48, 513, 16))
FAKE = 0x1000          # never dereferenced: every call below must be refused before it touches memory


def spec_of(h, w, batch=1, ct=3, z=64, loss=0):
    from carla_ppo_b200 import _lib
    base = _lib.VaeConfig(batch, ct, z, loss, _lib.FRAME_F32, _lib.FRAME_F32, 1.0 / 255, 1.0, 0.0, 1.0)
    return _lib.VaeSpec(base, h, w)


def spec_layout(lib, spec):
    n = lib.cpb_vae_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
    assert lib.cpb_vae_spec_layout(C.byref(spec), offs, sizes, shapes, C.byref(total)) == 0, lib.cpb_last_error()
    return list(offs), list(sizes), list(shapes), total.value


def encoded(h, w):
    for _ in range(4):
        h, w = (h - 4) // 2 + 1, (w - 4) // 2 + 1
    return h, w


@pytest.mark.parametrize("ct", [3, 1])
def test_spec_layout_matches_the_oracle_at_every_frame_size(lib, ct):
    from oracle.vae_oracle import param_shapes
    n = lib.cpb_vae_num_tensors()
    names = [lib.cpb_vae_tensor_name(i).decode() for i in range(n)]
    for h in SIDES:
        for w in SIDES:
            z = 64 if (h + w) % 32 == 0 else 100
            offs, sizes, shapes, total = spec_layout(lib, spec_of(h, w, ct=ct, z=z))
            ref = param_shapes((h, w, 3), ct, z)
            assert names == list(ref.keys())
            spans = []
            for i, name in enumerate(names):
                assert tuple(s for s in shapes[4 * i:4 * i + 4] if s > 0) == ref[name], (h, w, name)
                assert sizes[i] == int(np.prod(ref[name]))
                assert offs[i] % 64 == 0
                spans.append((offs[i], offs[i] + sizes[i]))
            spans.sort()
            assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), (h, w)
            assert spans[-1][1] <= total and total % 64 == 0
            h4, w4 = encoded(h, w)
            assert ref["mean/kernel"] == (h4 * w4 * 256, z)
            # the decoder maps [H4, W4] back to exactly [H, W] (reference vae/models.py:265)
            hh, ww = h4, w4
            for k in (4, 4, 5, 4):
                hh, ww = (hh - 1) * 2 + k, (ww - 1) * 2 + k
            assert (hh, ww) == (h, w)


@pytest.mark.parametrize("ct", [3, 1])
def test_legacy_entry_points_are_the_spec_at_80x160(lib, ct):
    n = lib.cpb_vae_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))(); total = C.c_int64()
    for z in (4, 64, 100):
        assert lib.cpb_vae_layout(ct, z, offs, sizes, shapes, C.byref(total)) == 0
        assert (list(offs), list(sizes), list(shapes), total.value) == spec_layout(lib, spec_of(80, 160, ct=ct, z=z))
        for batch in (1, 3, 257, 4096):
            for mode in (0, 1, 2):
                legacy = lib.cpb_vae_workspace_bytes(batch, ct, z, mode)
                assert legacy > 0
                assert lib.cpb_vae_spec_workspace_bytes(C.byref(spec_of(80, 160, batch, ct, z)), mode) == legacy
                cap = 18
                a = (C.c_int64 * cap)(); b = (C.c_int64 * cap)()
                assert lib.cpb_debug_vae_buffer_offsets(batch, ct, z, mode, a, cap) == cap
                assert lib.cpb_debug_vae_spec_buffer_offsets(C.byref(spec_of(80, 160, batch, ct, z)), mode, b, cap) == cap
                assert list(a) == list(b)
        cfg = spec_of(80, 160, 8, ct, z).base
        assert lib.cpb_vae_staging_bytes(C.byref(cfg)) == lib.cpb_vae_spec_staging_bytes(C.byref(spec_of(80, 160, 8, ct, z)))


def test_workspace_grows_with_the_frame(lib):
    small = lib.cpb_vae_spec_workspace_bytes(C.byref(spec_of(48, 48, 16)), 2)
    default = lib.cpb_vae_spec_workspace_bytes(C.byref(spec_of(80, 160, 16)), 2)
    large = lib.cpb_vae_spec_workspace_bytes(C.byref(spec_of(512, 512, 16)), 2)
    assert 0 < small < default < large
    # staging: one source frame, one target frame (uint8 here) and the noise rows, each rounded up to 256 bytes, + 256
    from carla_ppo_b200 import _lib
    sp = spec_of(64, 128, 5, ct=1, z=64)
    sp.base.source_dtype = sp.base.target_dtype = _lib.FRAME_U8
    up = lambda v: (v + 255) // 256 * 256
    assert lib.cpb_vae_spec_staging_bytes(C.byref(sp)) == up(5 * 64 * 128 * 3) + up(5 * 64 * 128) + up(5 * 64 * 4) + 256


ILLEGAL = [(40, 160), (72, 160), (528, 160), (0, 160), (-16, 160), (80, 72), (80, 40), (80, 528), (80, 0), (80, -80),
           (81, 160), (80, 168)]


def _compute_calls(lib, sp):
    """Every spec compute entry point with pointers that must never be dereferenced."""
    from carla_ppo_b200 import _lib
    ppo = _lib.PpoConfig(); ppo.state_dim, ppo.num_actions, ppo.hidden1, ppo.hidden2 = 67, 2, 500, 300
    ws = 1 << 40
    s = C.byref(sp)
    return {
        "encode": lambda: lib.cpb_vae_spec_encode(s, FAKE, FAKE, FAKE, None, None, FAKE, ws, None),
        "decode": lambda: lib.cpb_vae_spec_decode(s, FAKE, FAKE, FAKE, FAKE, ws, None),
        "forward": lambda: lib.cpb_vae_spec_forward(s, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, None, None, None, FAKE, ws, None),
        "loss_grad": lambda: lib.cpb_vae_spec_loss_grad(s, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, ws, None),
        "train_step": lambda: lib.cpb_vae_spec_train_step(s, FAKE, FAKE, FAKE, FAKE, FAKE, 1e-4, FAKE, FAKE, FAKE, FAKE, None,
                                                          FAKE, ws, None),
        "train_step_host": lambda: lib.cpb_vae_spec_train_step_host(s, FAKE, FAKE, FAKE, FAKE, FAKE, 1e-4, FAKE, FAKE, FAKE, FAKE,
                                                                    None, FAKE, ws, FAKE, ws, None),
        "encode_predict": lambda: lib.cpb_vae_spec_encode_predict(s, FAKE, FAKE, FAKE, 3, C.byref(ppo), FAKE, None, FAKE, FAKE,
                                                                  FAKE, FAKE, None, FAKE, ws, FAKE, ws, None),
    }


@pytest.mark.parametrize("hw", ILLEGAL)
def test_illegal_frames_are_refused_before_touching_memory(lib, hw):
    h, w = hw
    sp = spec_of(h, w, batch=2)
    before = lib.cpb_launch_count()
    for name, call in _compute_calls(lib, sp).items():
        assert call() == -1, name
        assert b"multiple of 16 in [48, 512]" in lib.cpb_last_error(), name
    assert lib.cpb_vae_spec_layout(C.byref(sp), None, None, None, None) == -1
    assert b"frame %dx%d" % (h, w) in lib.cpb_last_error()
    assert lib.cpb_vae_spec_workspace_bytes(C.byref(sp), 2) == -1
    assert b"bad arguments" in lib.cpb_last_error()
    assert lib.cpb_vae_spec_staging_bytes(C.byref(sp)) == -1
    offs = (C.c_int64 * 18)()
    assert lib.cpb_debug_vae_spec_buffer_offsets(C.byref(sp), 2, offs, 18) == -1
    assert lib.cpb_launch_count() == before


def test_bad_channels_and_null_spec_are_refused(lib):
    for ct in (0, 2, 4):
        sp = spec_of(64, 128, batch=2, ct=ct)
        for name, call in _compute_calls(lib, sp).items():
            assert call() == -1, name
        assert lib.cpb_vae_spec_layout(C.byref(sp), None, None, None, None) == -1
        assert b"target_channels" in lib.cpb_last_error()
        assert lib.cpb_vae_spec_workspace_bytes(C.byref(sp), 0) == -1
    assert lib.cpb_vae_spec_layout(None, None, None, None, None) == -1
    assert lib.cpb_vae_spec_workspace_bytes(None, 0) == -1
    assert lib.cpb_vae_spec_encode(None, FAKE, FAKE, FAKE, None, None, FAKE, 1 << 40, None) == -1


def tc_bound(h, w):
    """The largest batch of math modes 1 and 2: B * H1 * W1 * 32 < 2^31 (conv1's output is the largest tensor-core operand)."""
    return ((1 << 31) - 1) // ((h // 2 - 1) * (w // 2 - 1) * 32)


def test_batch_bound_table():
    assert (tc_bound(80, 160), tc_bound(160, 320), tc_bound(512, 512)) == (21781, 5342, 1032)


@pytest.mark.parametrize("hw", [(80, 160), (160, 320), (512, 512), (48, 512)])
@pytest.mark.parametrize("mode", [1, 2])
def test_batch_over_the_bound_is_refused_before_any_launch(lib, hw, mode):
    h, w = hw
    bound = tc_bound(h, w)
    with math_mode(lib, mode):
        before = lib.cpb_launch_count()
        for name, call in _compute_calls(lib, spec_of(h, w, batch=bound + 1)).items():
            assert call() == -4, name                                       # CPB_ERR_UNSUPPORTED
            assert (b"batch=%d is above %d" % (bound + 1, bound)) in lib.cpb_last_error(), name
        assert lib.cpb_launch_count() == before
        # the legacy entry points are the same code at 80x160
        if (h, w) == (80, 160):
            cfg = spec_of(80, 160, batch=bound + 1).base
            assert lib.cpb_vae_encode(C.byref(cfg), FAKE, FAKE, FAKE, None, None, FAKE, 1 << 40, None) == -4
        # at the bound the check passes: a zero-byte workspace is what stops the call (or the missing device here)
        sp = spec_of(h, w, batch=bound)
        assert lib.cpb_vae_spec_encode(C.byref(sp), FAKE, FAKE, FAKE, None, None, FAKE, 0, None) not in (0, -4)
        assert lib.cpb_launch_count() == before
        # the query calls take any batch: they do not depend on the math mode
        assert lib.cpb_vae_spec_workspace_bytes(C.byref(spec_of(h, w, batch=bound + 1)), 2) > 0


def test_mode_0_takes_batches_above_the_tensor_core_bound(lib):
    with math_mode(lib, 0):
        sp = spec_of(512, 512, batch=tc_bound(512, 512) + 1)
        assert lib.cpb_vae_spec_encode(C.byref(sp), FAKE, FAKE, FAKE, None, None, FAKE, 0, None) not in (0, -4)


@pytest.mark.parametrize("hw", [(48, 48), (64, 96), (112, 208)])
@pytest.mark.parametrize("ct", [3, 1])
def test_oracle_backward_matches_autograd_away_from_80x160(hw, ct):
    from oracle import vae_oracle as vo, torch_ref as tr
    h, w = hw
    z = 64 if ct == 3 else 100
    p = vo.glorot_init(h + w + ct, (h, w, 3), ct, z)
    rs = np.random.RandomState(h * w + ct)
    x = rs.rand(2, h, w, 3)
    y = x if ct == 3 else rs.rand(2, h, w, 1)
    eps = rs.randn(2, z)
    for loss, beta, tol in (("mse", 1.0, 0.0), ("bce", 1.0, 0.0), ("bce_v2", 3.0, 0.4)):
        a = vo.loss_and_grads(p, x, y, eps, loss, beta, tol)
        b = tr.vae_loss_and_grads(p, x, y, eps, loss, beta, tol)
        assert a["logits"].shape == (2, h, w, ct)
        assert abs(a["recon"] - b["recon"]) < 1e-10 * abs(b["recon"])
        assert abs(a["kl"] - b["kl"]) < 1e-10 * max(abs(b["kl"]), 1)
        assert set(a["grads"]) == set(b["grads"]) and len(a["grads"]) == 22
        for k in a["grads"]:
            assert rel_l2(a["grads"][k], b["grads"][k]) < 1e-10, (hw, ct, loss, k)


def test_constructor_rule(tmp_path):
    from carla_ppo_b200.vae.models import ConvVAE, MlpVAE
    for h, w in ((48, 48), (64, 128), (512, 48), (48, 512), (512, 512), (96, 64)):
        for ct in (3, 1):
            v = ConvVAE((h, w, 3), target_shape=(h, w, ct), z_dim=64, model_dir=str(tmp_path / ("ok%d_%d_%d" % (h, w, ct))))
            assert v.source_shape == (h, w, 3) and v.target_shape == (h, w, ct)
            assert v.encoded_shape == encoded(h, w) + (256,)
    for h, w in ILLEGAL:
        with pytest.raises(ValueError, match=r"frame %dx%d: height and width must each be a multiple of 16 in \[48, 512\]" % (h, w)):
            ConvVAE((h, w, 3), model_dir=str(tmp_path / "bad"))
    for bad_target in ((64, 128, 2), (64, 64, 3), (128, 64, 3)):
        with pytest.raises(ValueError, match="target_shape"):
            ConvVAE((64, 128, 3), target_shape=bad_target, model_dir=str(tmp_path / "bad"))
    with pytest.raises(ValueError, match="source_shape"):
        ConvVAE((64, 128, 1), target_shape=(64, 128, 1), model_dir=str(tmp_path / "bad"))
    # the target defaults to the source at the reference's 80x160 only; any other frame names its target
    assert ConvVAE((80, 160, 3), model_dir=str(tmp_path / "d")).target_shape == (80, 160, 3)
    assert ConvVAE(np.array([80, 160, 3]), model_dir=str(tmp_path / "d")).target_shape == (80, 160, 3)
    for h, w in ((64, 64), (64, 128), (48, 512)):
        with pytest.raises(ValueError, match=r"ConvVAE at frame %dx%d: give target_shape" % (h, w)):
            ConvVAE((h, w, 3), model_dir=str(tmp_path / "t"))
    # the MlpVAE keeps the reference's 80x160 input
    MlpVAE((80, 160, 3), z_dim=64, model_dir=str(tmp_path / "mlp"))
    for shape in ((64, 128, 3), (48, 48, 3), (160, 80, 3)):
        with pytest.raises(ValueError, match="MlpVAE is built for source_shape"):
            MlpVAE(shape, model_dir=str(tmp_path / "mlpbad"))


def test_recorded_source_shape(tmp_path):
    from carla_ppo_b200.vae.models import recorded_source_shape
    d = tmp_path / "checkpoints"
    d.mkdir()
    assert recorded_source_shape(str(d)) is None
    np.savez(str(d / "model.ckpt-3.npz"), **{"vae/step_idx": np.int32(3), "vae/source_shape": np.array([64, 128, 3], np.int32)})
    (d / "checkpoint").write_text('model_checkpoint_path: "model.ckpt-3"\nall_model_checkpoint_paths: "model.ckpt-3"\n')
    assert recorded_source_shape(str(d)) == (64, 128, 3)
    np.savez(str(d / "model.ckpt-4.npz"), **{"vae/step_idx": np.int32(4)})        # written before the shape was recorded
    (d / "checkpoint").write_text('model_checkpoint_path: "model.ckpt-4"\n')
    assert recorded_source_shape(str(d)) is None
