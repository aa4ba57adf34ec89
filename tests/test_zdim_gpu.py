"""GPU tests of latent sizes that are not multiples of 64 (z_dim 16, 32, 100): the library pads the latent to
64 * ceil(z / 64) columns inside the workspace and keeps the reference's [B, z] / TF-shaped boundary.

Gates are those of tests/test_vae_gpu.py: forward tensors, losses and parameters after Adam within 1e-5 relative L2 of
the float64 oracle (Adam: or 1.5 x the float32 CPU restatement's own error, as test_train_steps_follow_oracle_trajectory),
gradients within max(1e-5, 2 x the float32 CPU restatement's error); math mode 2 against the TF32 restatement with the
gates of tests/test_tf32_gpu.py."""
import os

import numpy as np
import pytest

import harness
import tf32_oracle
from harness import conv_relu_masks, dev, lib, library_state, make_conv_vae  # noqa: F401
from helpers import committed_frames, rel_l2
from ppo_cases import train_params
from vae_checks import grad_check, shift_away_from_zero

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-5
_WEIGHTS = {}


@pytest.fixture(scope="module")
def oracle():
    from oracle import vae_oracle
    return vae_oracle


@pytest.fixture(params=[1, 0], ids=["tc3xtf32", "simt"])
def math_mode(request, lib):
    with harness.math_mode(lib, request.param):
        yield request.param


def inputs(n, z, seed=0):
    x = np.random.RandomState(seed).rand(n, 80, 160, 3).astype(np.float32)
    eps = np.random.RandomState(seed + 1).randn(n, z).astype(np.float32)
    return x, eps


def weights(oracle, z):
    """Glorot kernels with small non-zero biases, then shifted off the ReLU kinks on inputs(2, z) like
    tests/test_vae_gpu.py::test_gradients_against_the_oracles_own_relu_masks."""
    if z not in _WEIGHTS:
        w = oracle.glorot_init(z, z_dim=z)
        for k in w:
            if k.endswith("bias"):
                w[k] = (0.05 * np.random.RandomState(len(k)).randn(*w[k].shape)).astype(np.float32)
        x, eps = inputs(2, z)
        _WEIGHTS[z] = shift_away_from_zero(oracle, w, x, eps, margin=2e-5)
    return {k: v.copy() for k, v in _WEIGHTS[z].items()}


@pytest.mark.parametrize("z", [16, 32, 100])
def test_conv_vae_forward_gradients_and_adam_match_oracle(tmp_path, oracle, math_mode, z):
    import torch
    from oracle import torch_ref
    w = weights(oracle, z)
    vae = make_conv_vae(tmp_path, w, z=z, learning_rate=1e-4)
    # forward: every tensor that crosses the boundary at [B, z]
    x, eps = inputs(6, z, seed=3)
    out = vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps), want_reconstruction=True, want_latents=True)
    ref = oracle.loss_and_grads(w, x, x, eps, "mse", want_grads=False)
    for k in ("mean", "logvar", "z"):
        assert out[k].shape == (6, z)
        assert rel_l2(out[k].cpu().numpy(), ref[k]) < FWD_TOL, k
    rec = out["reconstruction"].cpu().numpy().reshape(6, 80, 160, 3)
    assert rel_l2(rec, oracle.sigmoid(ref["logits"])) < FWD_TOL
    losses = out["losses"].cpu().numpy()
    assert abs(losses[0] - ref["recon"]) / ref["recon"] < FWD_TOL
    assert abs(losses[1] - ref["kl"]) < FWD_TOL          # KL ~ 0.1-0.9 here, a cancelling sum: absolute gate, as for glorot0
    # all 22 gradients, on the inputs the biases were shifted for
    x2, eps2 = inputs(2, z)
    grad_check(vae, oracle, w, x2, x2, eps2, "mse", floor=FWD_TOL)
    # two Adam steps
    p64 = {k: v.astype(np.float64) for k, v in w.items()}
    st = oracle.adam_init_state(p64)
    cpu32 = torch_ref.TorchVAETrainer(w, lr=1e-4)
    for step in range(2):
        xs, es = inputs(4, z, seed=20 + 2 * step)
        got_l = vae.train_step_device(dev(vae, xs), dev(vae, xs), dev(vae, es)).cpu().numpy()
        recon, _ = oracle.train_step(p64, st, xs, xs, es, lr=1e-4)
        cpu32.step(torch.from_numpy(xs), torch.from_numpy(xs), torch.from_numpy(es))
        assert abs(got_l[0] - recon) / recon < FWD_TOL
        got = vae.get_weights()
        for name in p64:
            assert got[name].shape == w[name].shape
            c32 = cpu32.p[name].detach().numpy()
            assert rel_l2(got[name], p64[name]) < max(FWD_TOL, 1.5 * rel_l2(c32, p64[name])), (step, name)


def test_kl_tolerance_floor_at_z32(tmp_path, oracle, math_mode):
    """kl_tolerance > 0 with the floor (kl_tolerance * z, the REAL z) active on some rows only: KL value and gradients."""
    z = 32
    w = weights(oracle, z)
    w["mean/bias"] = np.linspace(-1.5, 1.5, z).astype(np.float32)
    x, eps = inputs(2, z)
    ref = oracle.loss_and_grads(w, x, x, eps, "mse", want_grads=False)
    rows = -0.5 * np.sum(1 + ref["logvar"] - ref["mean"] ** 2 - np.exp(ref["logvar"]), axis=1)
    tol = float(rows.mean()) / z                      # floor between the two rows
    assert (rows < tol * z).any() and (rows > tol * z).any()
    vae = make_conv_vae(tmp_path, w, z=z, kl_tolerance=tol)
    out = vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps))["losses"].cpu().numpy()
    ref = oracle.loss_and_grads(w, x, x, eps, "mse", 1.0, tol, want_grads=False)
    assert abs(out[1] - ref["kl"]) / ref["kl"] < FWD_TOL
    grad_check(vae, oracle, w, x, x, eps, "mse", kl_tolerance=tol, floor=FWD_TOL)


def test_mlp_vae_at_z32_matches_oracle(tmp_path, oracle):
    """As tests/test_vae_gpu.py::test_mlp_vae_matches_oracle, at z = 32 (the MlpVAE is SIMT in every math mode)."""
    import torch
    from carla_ppo_b200.vae.models import MlpVAE
    from oracle import torch_ref
    z = 32
    w = oracle.mlp_glorot_init(1, z_dim=z)
    for k in w:
        if k.endswith("bias"):
            w[k] = (0.05 * np.random.RandomState(len(k)).randn(*w[k].shape)).astype(np.float32)
    vae = MlpVAE(source_shape=(80, 160, 3), z_dim=z, loss_fn="bce", model_dir=str(tmp_path / "mlp_zdim32"), seed=0)
    vae.init_session(init_logging=False)
    vae.set_weights(w)
    x, eps = inputs(6, z)
    out = vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps), want_reconstruction=True, want_latents=True)
    ref = oracle.mlp_loss_and_grads(w, x, x, eps, "bce")
    for k in ("mean", "logvar", "z"):
        assert out[k].shape == (6, z) and rel_l2(out[k].cpu().numpy(), ref[k]) < FWD_TOL, k
    assert rel_l2(out["reconstruction"].cpu().numpy(), oracle.sigmoid(ref["logits"])) < FWD_TOL
    losses = out["losses"].cpu().numpy()
    assert abs(losses[0] - ref["recon"]) / ref["recon"] < FWD_TOL and abs(losses[1] - ref["kl"]) / ref["kl"] < FWD_TOL
    vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
    got = vae.get_grads()
    ref32 = torch_ref.mlp_vae_loss_and_grads(w, x, x, eps, "bce", dtype=torch.float32)
    for name, g in ref["grads"].items():
        gate = max(FWD_TOL, 2.0 * rel_l2(ref32["grads"][name], g))
        assert rel_l2(got[name], g) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], g), gate)
    p64 = {k: v.astype(np.float64) for k, v in w.items()}
    st = oracle.adam_init_state(p64)
    for _ in range(2):
        vae.train_step(x, x, eps)
        oracle.mlp_train_step(p64, st, x, x, eps, lr=1e-4, loss_type="bce")
    gotw = vae.get_weights()
    for name in p64:
        assert rel_l2(gotw[name], p64[name]) < FWD_TOL, name
    mu = vae.encode(x[:2])
    assert mu.shape == (2, z)
    gen = vae.generate_from_latent(mu)
    assert gen.shape == (2, 38400)
    ref_gen = oracle.sigmoid(oracle.mlp_loss_and_grads(gotw, x[:2], x[:2], np.zeros((2, z)), "bce", want_grads=False)["logits"])
    mu_ref = oracle.mlp_loss_and_grads(gotw, x[:2], x[:2], np.zeros((2, z)), "bce", want_grads=False)["mean"]
    assert rel_l2(mu, mu_ref) < FWD_TOL and rel_l2(gen, ref_gen.reshape(2, -1)) < FWD_TOL
    assert vae.reconstruct(x[:1])[0].shape == (80, 160, 3)
    vae.save()
    from carla_ppo_b200 import vae_common
    again = vae_common.load_vae(str(tmp_path / "mlp_zdim32"))
    assert type(again).__name__ == "MlpVAE" and again.z_dim == z
    assert np.array_equal(again.encode(x[:2]), vae.encode(x[:2]))


def test_tf32_mode_at_z32_within_twice_the_tf32_restatement(tmp_path, lib, oracle):
    """Math mode 2 at z = 32: forward tensors, losses and all 22 gradients within max(1e-5, 2 x err_tf32) of float64,
    as tests/test_tf32_gpu.py::test_model_matches_float64_within_twice_the_tf32_restatement."""
    from carla_ppo_b200 import _lib
    z = 32
    w = weights(oracle, z)
    x, eps = inputs(8, z, seed=5)
    with harness.math_mode(lib, _lib.MATH_TF32):
        vae = make_conv_vae(tmp_path, w, z=z)
        out = vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps), want_reconstruction=True, want_latents=True)
        fwd = {k: out[k].cpu().numpy().astype(np.float64) for k in ("mean", "logvar", "z", "reconstruction")}
        vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
        got = vae.get_grads()
        losses = vae._losses.cpu().numpy().astype(np.float64)
        masks = conv_relu_masks(vae, 8)
    ref = oracle.loss_and_grads(w, x, x, eps, "mse", relu_masks=masks)
    t32 = tf32_oracle.loss_and_grads(w, x, x, eps, "mse", relu_masks=masks)
    for k in ("mean", "logvar", "z"):
        gate = max(FWD_TOL, 2.0 * rel_l2(t32[k], ref[k]))
        assert rel_l2(fwd[k], ref[k]) < gate, (k, rel_l2(fwd[k], ref[k]), gate)
    rec_ref = oracle.sigmoid(ref["logits"]).reshape(8, -1)
    gate = max(FWD_TOL, 2.0 * rel_l2(oracle.sigmoid(t32["logits"]).reshape(8, -1), rec_ref))
    assert rel_l2(fwd["reconstruction"], rec_ref) < gate
    for i, k in enumerate(("recon", "kl")):
        scale = 1.0 if k == "kl" else abs(ref[k])          # KL ~ 0.2: a cancelling sum, absolute errors
        gate = max(FWD_TOL, 2.0 * abs(t32[k] - ref[k]) / scale)
        assert abs(losses[i] - ref[k]) / scale < gate, (k, losses[i], ref[k], t32[k])
    for name, g in ref["grads"].items():
        gate = max(FWD_TOL, 2.0 * rel_l2(t32["grads"][name], g))
        assert rel_l2(got[name], g) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], g), gate)
    assert rel_l2(fwd["mean"], t32["mean"]) < rel_l2(fwd["mean"], ref["mean"])        # the single pass ran


def test_batch_invariance_and_reference_surface_at_z32(tmp_path, oracle, math_mode):
    """Encoding B frames == encoding its four quarters, bit for bit; encode() == forward_device()["mean"] bit for bit;
    decode / generate_from_latent / reconstruct have the reference shapes (and decode matches the oracle)."""
    import torch
    z = 32
    w = weights(oracle, z)
    vae = make_conv_vae(tmp_path, w, z=z, training=False)
    g = torch.Generator(device="cuda"); g.manual_seed(0)
    B = 1024
    x = torch.rand(B, 80, 160, 3, generator=g, device="cuda")
    full = vae.forward_device(x, x, None, want_latents=True)["mean"].clone()
    q = B // 4
    parts = [vae.forward_device(x[i * q:(i + 1) * q], x[i * q:(i + 1) * q], None, want_latents=True)["mean"].clone()
             for i in range(4)]
    assert full.shape == (B, z) and torch.equal(full, torch.cat(parts))
    frames = x[:5].cpu().numpy()
    mu = vae.encode(frames)
    assert mu.shape == (5, z) and mu.dtype == np.float32
    assert np.array_equal(mu, full[:5].cpu().numpy())
    gen = vae.generate_from_latent(mu)
    assert gen.shape == (5, 80 * 160 * 3)
    assert rel_l2(gen, oracle.decode({k: v.astype(np.float64) for k, v in w.items()}, mu.astype(np.float64))) < FWD_TOL
    rec = vae.reconstruct(frames[:3])
    assert len(rec) == 3 and rec[0].shape == (80, 160, 3)


def test_fused_actor_with_a_z32_vae(tmp_path, oracle):
    """train.py over the replay environment with a z = 32 VAE and a PPO of state_dim 35: the fused per-step call
    (cpb_encode_predict) and the unfused encode + PPO.predict produce the same trajectory and weights, bit for bit."""
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    rgb, _ = committed_frames()
    w = weights(oracle, 32)
    runs = []
    for tag, over in (("fused", {}), ("unfused", {"unfused": True})):
        env = ReplayEnv(rgb, episode_length=24, seed=0)
        vae = make_conv_vae(tmp_path, w, z=32, tag="vae_" + tag, training=False)
        model = train(train_params(tag, **over), restart=False, env=env, vae=vae, models_root=str(tmp_path / "models"),
                      interactive=False)
        assert model.state_dim == 35 and env.step_count > 0
        runs.append(model)
    a, b = runs
    wa, wb = a.get_weights(), b.get_weights()
    assert a.get_train_step_idx() == b.get_train_step_idx() > 0
    assert all(np.array_equal(wa[k], wb[k]) for k in wa)
    assert a.reward_history == b.reward_history


def test_save_and_load_vae_from_a_zdim32_directory(tmp_path, oracle):
    from carla_ppo_b200 import vae_common
    w = weights(oracle, 32)
    name = "rgb_bce_cnn_zdim32_beta1_kl_tolerance0.0_data"
    vae = make_conv_vae(tmp_path, w, z=32, tag=name, loss="bce")
    vae.save()
    again = vae_common.load_vae(str(tmp_path / name))
    assert type(again).__name__ == "ConvVAE" and again.z_dim == 32
    x, _ = inputs(3, 32)
    assert np.array_equal(again.encode(x), vae.encode(x))


def test_train_vae_cli_with_z_dim_32(tmp_path):
    from PIL import Image
    from carla_ppo_b200.vae import train_vae
    rgb, _ = committed_frames()
    data = tmp_path / "data"
    (data / "rgb").mkdir(parents=True)
    for i in range(24):
        Image.fromarray(rgb[i]).save(data / "rgb" / ("%d.png" % i))
    vae = train_vae.main(["--dataset", str(data), "--batch_size", "8", "--max_epochs", "1", "--loss_type", "mse",
                          "--z_dim", "32", "--models_root", str(tmp_path / "models"), "-restart"])
    assert vae.z_dim == 32 and "rgb_mse_cnn_zdim32_" in vae.model_dir
    assert vae.encode(rgb[:2]).shape == (2, 32)
    assert np.isfinite(vae.evaluate(rgb[:8], rgb[:8], 8)).all()
    assert any(f.endswith(".npz") for f in os.listdir(vae.checkpoint_dir))
