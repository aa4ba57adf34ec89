"""Pins of the oracle itself (CPU only): hand-derived backward vs torch autograd, the reference's own
artefacts (shipped checkpoints, frames, logged losses, Adam beta-powers), and -- when /root/reference is
present (build container) -- the reference's own compute_gae source and the full 1000-frame known-answer test."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest

from helpers import GOLDEN, committed_frames, kat, rel_l2, shipped_ppo, shipped_vae_weights

# The original project's source tree (TF graphs, checkpoints, frames, utils.py).  It is not part of this repository and is
# too large to store under tests/golden, so the tests marked with it run only where a copy sits at this path; everywhere
# else they skip by design.  What they check is also pinned by the committed fixtures the other tests in this module read.
REF = "/root/reference"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_vae_backward_matches_autograd():
    from oracle import vae_oracle as vo, torch_ref as tr
    p = vo.glorot_init(0)
    rs = np.random.RandomState(0)
    x = rs.rand(3, 80, 160, 3).astype(np.float32)
    eps = rs.randn(3, 64)
    for loss, beta, tol in (("mse", 1.0, 0.0), ("bce", 1.0, 0.0), ("bce_v2", 3.0, 0.4)):
        a = vo.loss_and_grads(p, x, x, eps, loss, beta, tol)
        b = tr.vae_loss_and_grads(p, x, x, eps, loss, beta, tol)
        assert abs(a["recon"] - b["recon"]) < 1e-9 * abs(b["recon"])
        assert abs(a["kl"] - b["kl"]) < 1e-9 * max(abs(b["kl"]), 1)
        for k in a["grads"]:
            assert rel_l2(a["grads"][k], b["grads"][k]) < 1e-10, (loss, k)


def test_vae_segmentation_target_backward():
    from oracle import vae_oracle as vo, torch_ref as tr
    p = vo.glorot_init(1, target_channels=1)
    rs = np.random.RandomState(1)
    x = rs.rand(2, 80, 160, 3); y = rs.rand(2, 80, 160, 1); eps = rs.randn(2, 64)
    a = vo.loss_and_grads(p, x, y, eps, "bce")
    b = tr.vae_loss_and_grads(p, x, y, eps, "bce")
    assert a["logits"].shape == (2, 80, 160, 1)
    for k in a["grads"]:
        assert rel_l2(a["grads"][k], b["grads"][k]) < 1e-10, k


def test_known_answer_committed_frames_vs_logged_losses():
    """KAT-1 on the committed subset: shipped ckpt-232 + 128 shipped frames -> BCE recon within 1 % of the
    reference's logged 22 327-22 415 and KL within 5 % of 96.5 (stochastic z => statistical)."""
    from oracle import vae_oracle as vo
    w, _ = shipped_vae_weights()
    rgb, _ = committed_frames()
    x = rgb.astype(np.float32) / 255.0
    eps = np.random.RandomState(7).randn(len(x), 64)
    out = vo.loss_and_grads(w, x, x, eps, "bce", want_grads=False)
    k = kat()
    assert abs(out["recon"] - k["rgb232_bce_on_committed_frames"]["recon"]) < 1e-6
    logged = [v for _, v in k["logged"]["val"]["vae/reconstruction_loss"]] + [v for _, v in k["logged"]["train"]["vae/reconstruction_loss"]]
    assert min(logged) * 0.99 < out["recon"] < max(logged) * 1.01
    logged_kl = np.mean([v for _, v in k["logged"]["train"]["vae/kl_loss"]])
    assert abs(out["kl"] - logged_kl) / logged_kl < 0.05


def test_shipped_adam_state_is_consistent_with_tf_adam_form():
    """beta2_power = 0.999^(steps+1) with 90 steps/epoch (cross-checks the power-after-step convention), and the
    shipped m/v slots are plausible EMA states (v >= 0, |m| <= sqrt(v)/sqrt(1-beta2)-ish)."""
    _, z = shipped_vae_weights()
    b2p = float(z["beta2_power"]); b1p = float(z["beta1_power"])
    steps = np.log(b2p) / np.log(0.999) - 1
    assert abs(steps - round(steps)) < 0.5 and round(steps) % 90 == 0      # whole epochs of 90 minibatches
    assert b1p == 0.0 or b1p < 1e-30
    v = z["adam_v/encoder/conv2/kernel"]
    assert (v >= 0).all()


def test_ppo_backward_matches_autograd_on_shipped_agent():
    from oracle import ppo_oracle as po, torch_ref as tr
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    assert max(np.abs(pol[k] - old[k]).max() for k in pol) < 2e-2          # they differ by one update (last 32-sample minibatch steps)
    rs = np.random.RandomState(0)
    s = rs.randn(48, 67); a = np.clip(rs.randn(48, 2), [-1, 0], [1, 1]); ret = rs.randn(48); adv = rs.randn(48)
    low, high = np.array([-1.0, 0.0]), np.array([1.0, 1.0])
    A = po.loss_and_grads(pol, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    B = tr.ppo_loss_and_grads(pol, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    assert abs(A["loss"] - B["loss"]) < 1e-10
    assert 0.5 < A["mean_ratio"] < 2.0
    for k in A["grads"]:
        assert rel_l2(A["grads"][k], B["grads"][k]) < 1e-10, k


def test_gae_lfilter_form_equals_recursion_and_is_not_reset_at_terminals():
    from oracle import ppo_oracle as po
    rs = np.random.RandomState(0)
    r = rs.rand(300); v = rs.randn(300); d = rs.rand(300) < 0.1
    a = po.compute_gae(r, v, 0.3, d, 0.99, 0.95)
    b = po.compute_gae_loop(r, v, 0.3, d, 0.99, 0.95)
    assert a.dtype == np.float64 and np.abs(a - b).max() < 1e-12
    # a reset-at-terminal GAE differs: the reference's does NOT reset (SURVEY section 0, item 7)
    adv = np.zeros(300); acc = 0.0; vv = np.append(v, 0.3)
    for t in range(299, -1, -1):
        nd = 1.0 - d[t]
        acc = r[t] + nd * 0.99 * vv[t + 1] - vv[t] + 0.99 * 0.95 * nd * acc
        adv[t] = acc
    assert np.abs(adv - a).max() > 1e-3


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree only exists in the build container")
def test_compute_gae_against_the_reference_source_itself():
    """Import the reference's utils.py with tensorflow/cv2 stubbed out and run ITS compute_gae."""
    from oracle import ppo_oracle as po
    saved = {k: sys.modules.get(k) for k in ("tensorflow", "cv2")}
    sys.modules["tensorflow"] = types.SimpleNamespace(tanh=None)
    sys.modules["cv2"] = types.ModuleType("cv2")
    try:
        spec = importlib.util.spec_from_file_location("ref_utils", os.path.join(REF, "utils.py"))
        ref_utils = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref_utils)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    rs = np.random.RandomState(3)
    for T in (1, 17, 2048):
        r = list(rs.rand(T)); v = list(rs.randn(T).astype(np.float32)); d = list(rs.rand(T) < 0.05)
        ref = ref_utils.compute_gae(r, v, np.float32(0.25), d, 0.99, 0.95)
        got = po.compute_gae(r, v, np.float32(0.25), d, 0.99, 0.95)
        assert np.array_equal(ref, got)


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree only exists in the build container")
def test_known_answer_full_reference_fixtures():
    """KAT-1 (rgb ckpt-232) and KAT-2 (seg ckpt-255) on 400 shipped frames straight from /root/reference,
    through the TF-bundle reader: losses within 1 % / 5 % of the reference's event files."""
    from PIL import Image
    from carla_ppo_b200.tf_bundle import BundleReader, latest_checkpoint
    from oracle import vae_oracle as vo
    idx = np.random.RandomState(0).choice(10000, 400, replace=False)
    rgb = np.stack([np.asarray(Image.open("%s/vae/data/rgb/%d.png" % (REF, i)))[:, :, :3] for i in idx]).astype(np.float32) / 255
    seg = np.stack([np.asarray(Image.open("%s/vae/data/segmentation/%d.png" % (REF, i)))[:, :, :1] for i in idx]).astype(np.float32) / 12
    eps = np.random.RandomState(1).randn(400, 64)
    for tag, y, ct, recon_range, kl_ref in (("rgb", rgb, 3, (22327.0, 22415.0), 96.5), ("seg", seg, 1, (5792.0, 5923.0), 118.0)):
        ck = latest_checkpoint("%s/vae/models/%s_bce_cnn_zdim64_beta1_kl_tolerance0.0_data/checkpoints" % (REF, tag))
        r = BundleReader(ck)
        w = {n: r.get("vae/" + n) for n in vo.param_shapes(target_channels=ct)}
        out = vo.loss_and_grads(w, rgb, y, eps, "bce", want_grads=False)
        assert recon_range[0] * 0.99 < out["recon"] < recon_range[1] * 1.01, (tag, out["recon"])
        assert abs(out["kl"] - kl_ref) / kl_ref < 0.05, (tag, out["kl"])


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree only exists in the build container")
def test_committed_fixtures_equal_the_shipped_checkpoints():
    from carla_ppo_b200.tf_bundle import BundleReader
    w, z = shipped_vae_weights()
    r = BundleReader("%s/vae/models/rgb_bce_cnn_zdim64_beta1_kl_tolerance0.0_data/checkpoints/model.ckpt-232" % REF)
    for k in w:
        assert np.array_equal(w[k], r.get("vae/" + k))
    pol, _ = shipped_ppo("policy")
    r2 = BundleReader("%s/models/pretrained_agent/checkpoints/model.ckpt-705" % REF)
    for k in pol:
        assert np.array_equal(pol[k], r2.get("policy/" + k))
    assert int(r2.get("episode_counter")) == 705


# ----------------------------------------------------------------------------- reference-held graph constants
def _meta_constants():
    import json
    with open(os.path.join(GOLDEN, "meta_constants.json")) as f:
        return json.load(f)


def test_constants_pinned_to_the_shipped_graphs():
    """SURVEY section 8(c) item 5: the numeric constants of the reference's SHIPPED TF graphs (MetaGraphDefs written by
    TF 1.13.1, extracted into tests/golden/meta_constants.json by make_meta_constants.py) are the only reference-held
    pin of the PPO loss: the oracle's and the CUDA kernels' constants must be exactly these float32 values."""
    from oracle import ppo_oracle as po, vae_oracle as vo
    mc = _meta_constants()
    p, v = mc["ppo"]["constants"], mc["vae"]["constants"]
    assert po.LOG_SQRT_2PI == p["log_prob_const"] and po.ENTROPY_CONST == p["entropy_const"] and p["log_prob_half"] == -0.5
    # clip bounds: Python 1 -/+ 0.2 rounded to float32 (what the oracle uses) ...
    assert float(np.float32(1.0 - 0.2)) == p["clip_low"] and float(np.float32(1.0 + 0.2)) == p["clip_high"]
    # ... and what the CUDA head kernel computes in float32 from eps_clip = 0.2f (ppo_device.cuh: 1.f -/+ a.eps_clip)
    assert float(np.float32(1) - np.float32(0.2)) == p["clip_low"] and float(np.float32(1) + np.float32(0.2)) == p["clip_high"]
    assert float(np.float32(0.01)) == p["entropy_scale"] and p["value_scale"] == 1.0
    assert p["mean_affine_add"] == 1.0 and p["mean_affine_div"] == 2.0        # mu = low + (tanh + 1)/2 * (high - low)
    for c in (p, v):
        assert vo.ADAM_BETA1 == c["adam_beta1"] == c["beta1_power_init"]
        assert vo.ADAM_BETA2 == c["adam_beta2"] == c["beta2_power_init"]
        assert vo.ADAM_EPS == c["adam_epsilon"]
        assert float(np.float32(1e-4)) == c["learning_rate"]
    assert v["kl_minus_half"] == -0.5 and v["kl_one"] == 1.0 and v["reparam_half"] == 0.5
    assert v["range_low"] == 0.0 and v["range_high"] == 1.0 and v["beta"] == 1.0
    # the tie rule of tf.minimum's gradient (LessEqual + Select: ties go to the UNclipped branch) -- what
    # ppo_oracle.loss_and_grads ("first = unclipped <= clipped") and ppo_head_kernel implement
    assert mc["ppo"]["surrogate"]["min_grad_select"] == ["LessEqual", "Select"]
    assert mc["ppo"]["surrogate"]["Minimum_inputs"] == ["mul", "mul_1"]
    # layer semantics the restatement assumes (NHWC, VALID, stride 2, no dilation; transposed conv = Conv2DBackpropInput)
    for name, op in mc["vae"]["conv_ops"].items():
        assert op["strides"] == [1, 2, 2, 1] and op["padding"] == "VALID" and op["data_format"] == "NHWC" and op["dilations"] == [1, 1, 1, 1]
        assert op["op"] == ("Conv2D" if "encoder" in name else "Conv2DBackpropInput")
    for need in ("Conv2DBackpropFilter", "Conv2DBackpropInput", "Conv2D", "BiasAddGrad", "ReluGrad", "MatMul", "AddN"):
        assert need in mc["vae"]["gradient_ops"]
    # variable shapes of both graphs == the oracle's parameter tables (the rgb VAE; and the seg VAE copy inside the agent graph)
    for name, shape in vo.param_shapes(target_channels=3).items():
        assert tuple(mc["vae"]["variables"]["vae/" + name]) == shape, name
    for name, shape in vo.param_shapes(target_channels=1).items():
        assert tuple(mc["ppo"]["variables"]["vae/" + name]) == shape, name
    for name, shape in po.param_shapes().items():
        assert tuple(mc["ppo"]["variables"]["policy/" + name]) == shape == tuple(mc["ppo"]["variables"]["policy_old/" + name])


def test_cuda_device_code_uses_the_pinned_constants():
    """The PPO device code (ppo_device.cuh, which both learn paths compile) spells the same literals (grep-level check; the
    GPU tests check the numerics)."""
    mc = _meta_constants()["ppo"]["constants"]
    src = open(os.path.join(ROOT, "carla_ppo_b200", "csrc", "ppo_device.cuh")).read()
    assert ("kLogSqrt2Pi = %sf" % repr(mc["log_prob_const"])) in src
    assert ("kEntropyConst = %sf" % repr(mc["entropy_const"])) in src
    assert "unclipped <= clipped" in src


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree only exists in the build container")
def test_meta_constants_file_equals_the_shipped_graphs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_meta_constants", os.path.join(GOLDEN, "make_meta_constants.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.extract() == _meta_constants()


# ----------------------------------------------------------------------------- TF-V2 bundle writer
def test_tf_bundle_writer_round_trip(tmp_path):
    from carla_ppo_b200 import tf_bundle as tb
    rs = np.random.RandomState(0)
    tensors = {"vae/encoder/conv1/kernel": rs.randn(4, 4, 3, 32).astype(np.float32), "vae/step_idx": np.int32(7),
               "beta1_power": np.float32(0.5), "a/b": np.arange(10, dtype=np.int64), "z": rs.randn(3, 5)}
    tb.write_bundle(str(tmp_path / "model.ckpt-7"), tensors)
    got = tb.BundleReader(str(tmp_path / "model.ckpt-7")).all()
    assert set(got) == set(tensors)
    for k, v in tensors.items():
        assert got[k].dtype == np.asarray(v).dtype and got[k].shape == np.asarray(v).shape and np.array_equal(got[k], v), k
    assert tb.verify_bundle_crcs(str(tmp_path / "model.ckpt-7")) == len(tensors)
    assert tb.crc32c(b"123456789") == 0xE3069283                      # the CRC-32C check value


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree only exists in the build container")
def test_tf_bundle_crc_and_entries_pinned_to_a_shipped_checkpoint(tmp_path):
    """The writer's format code against a file TF itself wrote: every stored crc32c of the shipped agent checkpoint
    verifies with this implementation, and re-writing its tensors reproduces each entry's dtype/shape/size/crc."""
    from carla_ppo_b200 import tf_bundle as tb
    prefix = "%s/models/pretrained_agent/checkpoints/model.ckpt-705" % REF
    assert tb.verify_bundle_crcs(prefix) == 80
    small = {k: v for k, v in tb.BundleReader(prefix).all().items() if v.size < 40000}
    tb.write_bundle(str(tmp_path / "x"), small)
    a, b = tb.BundleReader(prefix), tb.BundleReader(str(tmp_path / "x"))
    for k in small:
        assert a.entries[k][:2] == b.entries[k][:2] and a.entries[k][3] == b.entries[k][3]


def test_mlp_vae_backward_matches_autograd():
    """MlpVAE (vae/models.py:271-299): hand-derived backward of the oracle vs torch autograd, all three losses."""
    from oracle import vae_oracle as vo, torch_ref as tr
    kw = dict(encoder_sizes=(64, 32), decoder_sizes=(32, 64))
    p = vo.mlp_glorot_init(3, **kw)
    shapes = vo.mlp_param_shapes()
    assert shapes["encoder/dense/kernel"] == (38400, 512) and shapes["decoder/dense_2/kernel"] == (512, 38400) and len(shapes) == 14
    rs = np.random.RandomState(0)
    x = rs.rand(3, 80, 160, 3).astype(np.float32); eps = rs.randn(3, 64)
    for loss, beta, tol in (("mse", 1.0, 0.0), ("bce", 2.0, 0.0), ("bce_v2", 1.0, 0.3)):
        a = vo.mlp_loss_and_grads(p, x, x, eps, loss, beta, tol)
        b = tr.mlp_vae_loss_and_grads(p, x, x, eps, loss, beta, tol)
        assert abs(a["recon"] - b["recon"]) < 1e-9 * abs(b["recon"]) and abs(a["kl"] - b["kl"]) < 1e-9 * max(abs(b["kl"]), 1)
        for k in a["grads"]:
            assert rel_l2(a["grads"][k], b["grads"][k]) < 1e-10, (loss, k)
