"""GPU tests of the glue either side of the hot path: vae_common (reference vae_common.py:6-62), and -- further down --
the re-authored train.py / run_eval.py loop over the offline replay environment."""
import os
import types

import numpy as np
import pytest

from helpers import committed_frames, rel_l2, shipped_vae_weights
from ppo_cases import shipped_vae, train_params

pytestmark = pytest.mark.gpu

RGB_DIR = "rgb_bce_cnn_zdim64_beta1_kl_tolerance0.0_data"


def lay_outshipped_vae(root):
    """Writes the shipped rgb checkpoint-232 (committed golden npz) as a TF-V2 tensor bundle under the reference's
    directory convention vae/models/<name>/checkpoints/model.ckpt-232.* + the ``checkpoint`` state file."""
    from carla_ppo_b200.tf_bundle import write_bundle
    w, z = shipped_vae_weights()
    ck = os.path.join(root, "vae", "models", RGB_DIR, "checkpoints")
    os.makedirs(ck)
    blob = {"vae/" + k: v for k, v in w.items()}
    blob["vae/step_idx"] = np.int32(232)
    blob["vae/beta1_power"] = np.float32(z["beta1_power"]); blob["vae/beta2_power"] = np.float32(z["beta2_power"])
    write_bundle(os.path.join(ck, "model.ckpt-232"), blob)
    with open(os.path.join(ck, "checkpoint"), "w") as f:
        f.write('model_checkpoint_path: "model.ckpt-232"\nall_model_checkpoint_paths: "model.ckpt-232"\n')
    return os.path.join(root, "vae", "models", RGB_DIR)


class FakeVehicle:
    def __init__(self, steer, throttle, speed):
        self.control = types.SimpleNamespace(steer=steer, throttle=throttle)
        self._speed = speed

    def get_speed(self):
        return self._speed

    def get_forward_vector(self):
        return types.SimpleNamespace(x=0.6, y=0.8, z=0.0)


def test_vae_common_load_and_encode_state(tmp_path):
    """load_vae parses z_dim / model type / target depth from the directory name and restores the TF-V2 bundle;
    create_encode_state_fn(env) = [VAE mean of the frame | steer, throttle, speed (| forward vector)], float64, for both
    uint8 observations and preprocess_frame()'d float observations (reference vae_common.py:6-62)."""
    from carla_ppo_b200 import vae_common
    from oracle import vae_oracle as vo
    model_dir = lay_outshipped_vae(str(tmp_path))
    vae = vae_common.load_vae(model_dir, z_dim=None, model_type=None)
    assert vae.z_dim == 64 and vae.target_shape == (80, 160, 3) and vae.training is False
    assert vae.get_step_idx() == 232
    w = shipped_vae_weights()[0]
    got = vae.get_weights()
    assert all(np.array_equal(got[k], w[k]) for k in w)

    rgb, _ = committed_frames()
    env = types.SimpleNamespace(observation=rgb[3], vehicle=FakeVehicle(0.25, 0.5, 7.5))
    fn = vae_common.create_encode_state_fn(vae, ["steer", "throttle", "speed"])
    state = fn(env)
    assert state.shape == (67,) and state.dtype == np.float64          # np.append upcasts (vae_common.py:61)
    p64 = {k: v.astype(np.float64) for k, v in w.items()}
    mu, _ = vo.encode(p64, vae_common.preprocess_frame(rgb[3:4]).astype(np.float64))
    assert rel_l2(state[:64], mu[0]) < 1e-5
    assert np.array_equal(state[64:], [0.25, 0.5, 7.5])
    # a float observation holding raw 0..255 pixel values goes through preprocess_frame (/255) like the reference's
    env_f = types.SimpleNamespace(observation=rgb[3].astype(np.float32), vehicle=env.vehicle)
    assert rel_l2(fn(env_f)[:64], mu[0]) < 1e-5
    fn4 = vae_common.create_encode_state_fn(vae, ["steer", "throttle", "speed", "orientation"])
    s4 = fn4(env)
    assert s4.shape == (70,) and np.allclose(s4[67:], [0.6, 0.8, 0.0])
    with pytest.raises(Exception, match="Failed to load VAE"):
        vae_common.load_vae(str(tmp_path / "vae" / "models" / "seg_bce_cnn_zdim64_beta1_kl_tolerance0.0_data"))


def test_checkpoints_written_in_tf_format_round_trip(tmp_path):
    """save(tf_format=True) writes a TF-V2 bundle (what the reference's saver.restore reads); load_latest_checkpoint
    restores weights, Adam slots, beta powers and step_idx from it."""
    from carla_ppo_b200.vae.models import ConvVAE
    from carla_ppo_b200.tf_bundle import BundleReader, verify_bundle_crcs
    w = shipped_vae_weights()[0]
    vae = ConvVAE((80, 160, 3), z_dim=64, loss_fn="mse", model_dir=str(tmp_path / "m"), seed=0)
    vae.init_session(init_logging=False)
    vae.set_weights(w)
    rgb, _ = committed_frames()
    vae.train_step(rgb[:4], rgb[:4], np.random.RandomState(0).randn(4, 64).astype(np.float32))
    vae.step_idx = 5
    vae.save(tf_format=True)
    prefix = os.path.join(vae.checkpoint_dir, "model.ckpt-5")
    assert verify_bundle_crcs(prefix) == 22 * 3 + 3
    names = BundleReader(prefix).keys()
    assert "vae/vae/encoder/conv1/kernel/Adam_1" in names and "vae/beta2_power" in names
    b = ConvVAE((80, 160, 3), z_dim=64, loss_fn="mse", model_dir=str(tmp_path / "m"), seed=1)
    b.init_session(init_logging=False)
    assert b.load_latest_checkpoint() is True and b.get_step_idx() == 5
    assert bool((b.params == vae.params).all()) and bool((b.adam_m == vae.adam_m).all()) and bool((b.adam_v == vae.adam_v).all())
    assert bool((b.adam_powers == vae.adam_powers).all())


# ----------------------------------------------------------------------------- train.py / run_eval.py over the replay env
def _run_training(tmp_path, tag, **over):
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    rgb, _ = committed_frames()
    env = ReplayEnv(rgb, episode_length=24, seed=0)
    vae = shipped_vae(tmp_path, tag)
    model = train(train_params(tag, **over), restart=False, env=env, vae=vae, models_root=str(tmp_path / "models"), interactive=False)
    return model, env


def test_train_loop_fused_unfused_and_reference_loop_agree(tmp_path):
    """train.py on the replay environment, 2 episodes (+ 2 evaluation episodes, a checkpoint): the fused per-step call
    (cpb_encode_predict) reproduces the two separate calls bit for bit, and PPO.learn reproduces the reference's Python
    minibatch loop over PPO.train (train.py:171-207)."""
    a, env_a = _run_training(tmp_path, "fused")
    b, _ = _run_training(tmp_path, "unfused", unfused=True)
    c, _ = _run_training(tmp_path, "refloop", unfused=True, reference_loop=True)
    wa, wb, wc = a.get_weights(), b.get_weights(), c.get_weights()
    assert a.get_episode_idx() == 2 and a.get_train_step_idx() == b.get_train_step_idx() == c.get_train_step_idx() > 0
    assert all(np.array_equal(wa[k], wb[k]) for k in wa)
    assert a.reward_history == b.reward_history
    for k in wa:
        assert rel_l2(wb[k], wc[k]) < 1e-6, k
    assert os.path.isfile(os.path.join(a.checkpoint_dir, "checkpoint"))             # the evaluation episode saved a checkpoint
    assert env_a.step_count > 0


def test_train_loop_matches_the_oracle_stepping_the_same_replay(tmp_path):
    """The whole RL loop -- encode_state (VAE mean), predict (sampled, clipped), env.step, GAE + PPO update -- against the
    float64 oracle driving an identical replay environment with the same noise and shuffle streams."""
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import ReplayEnv
    from oracle import ppo_oracle as po, vae_oracle as vo
    model, _ = _run_training(tmp_path, "gpu", eval_interval=1000)
    # ---- the same loop on the oracle
    rgb, _ = committed_frames()
    env = ReplayEnv(rgb, episode_length=24, seed=0)
    env.seed(0)
    np.random.seed(0)
    probe = PPO((67,), env.action_space, initial_std=0.4, model_dir=str(tmp_path / "probe"), seed=0)
    probe.init_session(init_logging=False)
    p = {k: v.astype(np.float64) for k, v in probe.get_weights().items()}         # the seed-0 initial weights train() started from
    st = vo.adam_init_state(p)
    noise_rng = np.random.RandomState(0)
    vw = {k: v.astype(np.float64) for k, v in shipped_vae_weights()[0].items()}
    low, high = env.action_space.low.astype(np.float64), env.action_space.high.astype(np.float64)

    def encode(e):
        mu, _ = vo.encode(vw, (e.observation.astype(np.float32) / 255.0)[None].astype(np.float64))
        return np.append(mu[0], [e.vehicle.control.steer, e.vehicle.control.throttle, e.vehicle.get_speed()])
    env.encode_state_fn = encode
    rewards_hist = []
    for episode in range(2):
        state, terminal, total = env.reset(), False, 0.0
        while not terminal:
            S, A, V, R, D = [], [], [], [], []
            for _ in range(16):
                act, val = po.predict(p, state, low, high, noise=noise_rng.randn(1, 2).astype(np.float32))
                new_state, r, terminal, _ = env.step(act)
                S.append(state); A.append(act); V.append(np.float32(val)); R.append(r); D.append(terminal)
                total += r
                state = new_state
                if terminal:
                    break
            _, last_v = po.predict(p, state, low, high, noise=noise_rng.randn(1, 2).astype(np.float32))
            perms = []
            for _ in range(2):
                idx = np.arange(len(R)); np.random.shuffle(idx); perms.append(idx)
            po.learn(p, st, np.array(S, np.float32), np.array(A, np.float32), V, R, D, np.float32(last_v), low, high, 0.99, 0.95, 1e-4, 0.2, 1.0, 0.01,
                     2, 8, perms)
        rewards_hist.append(total)
    got = model.get_weights()
    assert np.allclose(model.reward_history, rewards_hist, rtol=1e-5, atol=1e-7), (model.reward_history, rewards_hist)
    for k in p:
        assert rel_l2(got[k], p[k]) < 2e-5, "%s: %.3e" % (k, rel_l2(got[k], p[k]))


def test_run_eval_is_greedy_and_deterministic(tmp_path):
    from carla_ppo_b200.actor import FusedActor
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.run_eval import run_eval
    from carla_ppo_b200.vae_common import create_encode_state_fn
    from helpers import shipped_ppo
    rgb, _ = committed_frames()
    vae = shipped_vae(tmp_path, "eval")
    env = ReplayEnv(rgb, episode_length=20, seed=3)
    model = PPO((67,), env.action_space, model_dir=str(tmp_path / "agent"), seed=0)
    model.init_session(init_logging=False)
    pol, _ = shipped_ppo("policy")
    model.set_weights(pol, pol)
    env.encode_state_fn = create_encode_state_fn(vae, {"steer", "throttle", "speed"})
    r1 = run_eval(env, model)
    r2 = run_eval(env, model)
    actor = FusedActor(vae, model, {"steer", "throttle", "speed"})
    env.encode_state_fn = actor.encode_state_fn
    r3 = run_eval(env, model, actor=actor)
    assert r1 == r2 == r3 and env.step_count > 0
    assert actor.calls == env.step_count + 1                      # one fused call per reset / step, none extra for predict
