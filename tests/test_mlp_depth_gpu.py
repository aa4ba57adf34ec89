"""The MlpVAE at any depth on the device, and its math mode 2 (the five frame-wide products -- the first encoder
layer's forward and weight gradient, the output layer's forward, data gradient and weight gradient -- as ONE TF32 wgmma
pass with both operands rounded to nearest).  Pinned here:

  * modes 0 and 1: forward tensors, losses, every gradient and two Adam steps within max(1e-5, 2 x err_f32) of float64,
    err_f32 being the float32 restatement's distance from float64 on the same inputs (DESIGN section 4);
  * mode 2, also at the default two layers per side and at widths that are not multiples of 64: the same against the
    TF32 restatement (tests/mlp_depth_oracle.py with its rounding hook), the device closer to that restatement than to
    float64, each of the five frame-wide products on the device's own operands at the 2e-6 unit bar (B = 6 and the
    k-split B = 512), and batch independence;
  * mode 2 repeats bit for bit and leaves mode 1 bit-identical; a workspace sized in mode 1 is refused in mode 2
    before anything is launched; train_vae.py trains an MlpVAE in mode 2;
  * the default shape: the spec entry points and the legacy ones give bit-identical results and launch counts;
  * checkpoints of a deeper model reload bit for bit, in both formats;
  * the fused actor takes an MlpVAE and reproduces the unfused loop, and train.train runs with one."""
import ctypes as C
import os

import numpy as np
import pytest

import mlp_depth_oracle as mdo
from harness import dev, gate, lib, library_state, make_mlp, math_mode, mlp_relu_masks, mlp_workspace  # noqa: F401
from helpers import committed_frames, rel_l2
from tf32_oracle import round_tf32
from vae_checks import FWD_TOL, IN, UNIT_TOL, backward_products, forward_products, inputs, mlp_weights

SHAPES = {"1x1": ((512,), (512,)), "3x2": ((96, 256, 64), (160, 64))}
# mode 2 also at the default two layers per side, and at enc1 = 96 (32-wide tensor-core tiles on a width that is not a
# multiple of 64) with dec2 = 64 (the weight gradient with fewer than 128 rows, run as its transpose)
MODE2_SHAPES = dict(SHAPES, **{"2x2": ((512, 256), (256, 512)), "odd_widths": ((96, 64), (160, 64))})
CASES = {"z64_bce_rgb": (64, 3, "bce"), "z32_bce_rgb": (32, 3, "bce"), "z64_mse_seg": (64, 1, "mse")}
MEAS = ("steer", "throttle", "speed")


def _check_model(tmp_path, lib, shape, case, mode):
    """6 random frames through a model of `shape` in math `mode`: the device against float64, gated by the
    restatement of the mode (float32 in modes 0 and 1, the TF32 rounding hook in mode 2) on the same inputs."""
    from carla_ppo_b200 import _lib
    from oracle import vae_oracle as vo
    enc, dec = MODE2_SHAPES[shape]
    z, ct, loss = CASES[case]
    with math_mode(lib, mode):
        w = mlp_weights(1, target_channels=ct, z_dim=z, encoder_sizes=enc, decoder_sizes=dec)
        vae = make_mlp(tmp_path, w, enc, dec, loss, z, ct)
        x, y, eps = inputs(6, z, ct)
        out = vae.forward_device(dev(vae, x), dev(vae, y), dev(vae, eps), want_reconstruction=True, want_latents=True)
        fwd = {k: out[k].cpu().numpy().astype(np.float64) for k in ("mean", "logvar", "z", "reconstruction")}
        vae.loss_grad_device(dev(vae, x), dev(vae, y), dev(vae, eps))
        got = vae.get_grads()
        losses = vae._losses.cpu().numpy().astype(np.float64)
        masks = mlp_relu_masks(vae, 6)
        tc = mode == _lib.MATH_TF32

        def restated(params, **kw):      # the restatement the mode is gated by
            if tc:
                return mdo.loss_and_grads(params, x, y, eps, loss, tc_round=round_tf32, **kw)
            return mdo.loss_and_grads(params, x, y, eps, loss, dtype=np.float32, **kw)
        ref = mdo.loss_and_grads(w, x, y, eps, loss, relu_masks=masks)
        approx = restated(w, relu_masks=masks)
        for k in ("mean", "logvar", "z"):
            assert rel_l2(fwd[k], ref[k]) < gate(approx[k], ref[k], FWD_TOL), (k, rel_l2(fwd[k], ref[k]))
        rec = vo.sigmoid(ref["logits"])
        assert rel_l2(fwd["reconstruction"], rec) < gate(vo.sigmoid(approx["logits"]), rec, FWD_TOL)
        for i, k in enumerate(("recon", "kl")):
            scale = max(abs(ref[k]), 1.0)
            bar = max(FWD_TOL, 2.0 * abs(approx[k] - ref[k]) / scale)
            assert abs(losses[i] - ref[k]) / scale < bar, (k, losses[i], ref[k], approx[k])
        assert sorted(ref["grads"]) == sorted(vae._names) and len(vae._names) == 2 * (len(enc) + len(dec) + 3)
        for name, g in ref["grads"].items():
            bar = gate(approx["grads"][name], g, FWD_TOL)
            assert rel_l2(got[name], g) < bar, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], g), bar)
        if tc:                       # the single pass ran, with rounding to nearest
            assert rel_l2(fwd["mean"], approx["mean"]) < rel_l2(fwd["mean"], ref["mean"])
        # two Adam steps from the same weights
        p64 = {k: v.astype(np.float64) for k, v in w.items()}
        pr = {k: v.astype(np.float64) for k, v in w.items()}
        st64, str_ = vo.adam_init_state(p64), vo.adam_init_state(pr)
        for _ in range(2):
            vae.train_step(x, y, eps)
            mdo.train_step(p64, st64, x, y, eps, lr=1e-4, loss_type=loss)
            vo.adam_apply(pr, restated(pr)["grads"], str_, 1e-4)
        gotw = vae.get_weights()
        for name in p64:
            bar = gate(pr[name], p64[name], FWD_TOL)
            assert rel_l2(gotw[name], p64[name]) < bar, "%s: %.3e (gate %.3e)" % (name, rel_l2(gotw[name], p64[name]), bar)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_modes_0_and_1_match_float64_within_twice_the_float32_restatement(tmp_path, lib, shape, case, mode):
    _check_model(tmp_path, lib, shape, case, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("shape", sorted(MODE2_SHAPES))
def test_mode_2_matches_float64_within_twice_the_tf32_restatement(tmp_path, lib, shape, case):
    from carla_ppo_b200 import _lib
    _check_model(tmp_path, lib, shape, case, _lib.MATH_TF32)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [6, 512])
@pytest.mark.parametrize("shape", sorted(MODE2_SHAPES))
def test_mode_2_frame_wide_products_on_the_devices_own_inputs(tmp_path, lib, shape, batch):
    """First encoder layer forward and weight gradient, output layer forward and weight gradient against the
    fp32-summed product of the rounded operands; the output layer's data gradient through the weight gradient of the
    last hidden decoder layer, which the fp32 SIMT kernels compute from it."""
    from carla_ppo_b200 import _lib
    enc, dec = MODE2_SHAPES[shape]
    with math_mode(lib, _lib.MATH_TF32):
        w = mlp_weights(1, encoder_sizes=enc, decoder_sizes=dec)
        vae = make_mlp(tmp_path, w, enc, dec)
        x, _, eps = inputs(batch)
        vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps))
        assert np.array_equal(mlp_workspace(vae, batch, _lib.WS_FORWARD, {"x": IN})["x"], x.reshape(batch, -1))
        for what, err in forward_products(vae, w, batch).items():
            assert err < UNIT_TOL, (what, err)
        vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
        for what, err in backward_products(vae, w, batch).items():
            assert err < UNIT_TOL, (what, err)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(MODE2_SHAPES))
def test_mode_2_encoding_does_not_depend_on_the_batch(tmp_path, lib, shape):
    """The k-split and every tile choice are fixed by the layer shapes: 8 frames encode bit for bit as their quarters."""
    import torch
    from carla_ppo_b200 import _lib
    enc, dec = MODE2_SHAPES[shape]
    with math_mode(lib, _lib.MATH_TF32):
        vae = make_mlp(tmp_path, mlp_weights(1, encoder_sizes=enc, decoder_sizes=dec), enc, dec)
        x, _, _ = inputs(8)
        whole, whole_lv = vae.encode_device(dev(vae, x), return_logvar=True)
        parts = [vae.encode_device(dev(vae, x[i:i + 2]), return_logvar=True) for i in range(0, 8, 2)]
        assert torch.equal(whole, torch.cat([p[0] for p in parts])) and torch.equal(whole_lv, torch.cat([p[1] for p in parts]))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_default_shape_spec_and_legacy_entry_points_agree_bit_for_bit(tmp_path, lib, mode):
    import torch
    from carla_ppo_b200 import _lib
    with math_mode(lib, mode):
        vae = make_mlp(tmp_path, mlp_weights(), (512, 256), (256, 512))
        x, _, eps = inputs(8)
        xd, ed = dev(vae, x), dev(vae, eps)
        spec, cfg = vae._config(8), vae._mlp_config(8)
        need = lib.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), _lib.WS_TRAIN)
        assert need == lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), _lib.WS_TRAIN)
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        runs = []
        for fn, arg in ((lib.cpb_mlpvae_spec_loss_grad, spec), (lib.cpb_mlpvae_loss_grad, cfg)):
            grads = torch.full_like(vae.grads, float("nan"))
            losses = torch.empty(2, device="cuda")
            torch.cuda.synchronize()
            lib.cpb_reset_launch_count()
            _lib.check(fn(C.byref(arg), vae.params.data_ptr(), xd.data_ptr(), xd.data_ptr(), ed.data_ptr(), grads.data_ptr(),
                          losses.data_ptr(), None, ws.data_ptr(), need, _lib.current_stream_handle()))
            torch.cuda.synchronize()
            runs.append((grads, losses, lib.cpb_launch_count()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]) and runs[0][2] == runs[1][2] > 0
        mean = [torch.empty(8, 64, device="cuda") for _ in range(2)]
        ws_e = torch.empty(lib.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), _lib.WS_ENCODE), dtype=torch.uint8, device="cuda")
        _lib.check(lib.cpb_mlpvae_spec_encode(C.byref(spec), vae.params.data_ptr(), xd.data_ptr(), mean[0].data_ptr(), None, None,
                                              ws_e.data_ptr(), ws_e.numel(), _lib.current_stream_handle()))
        _lib.check(lib.cpb_mlpvae_encode(C.byref(cfg), vae.params.data_ptr(), xd.data_ptr(), mean[1].data_ptr(), None, None,
                                         ws_e.data_ptr(), ws_e.numel(), _lib.current_stream_handle()))
        assert torch.equal(mean[0], mean[1])


@pytest.mark.gpu
@pytest.mark.parametrize("tf_format", [False, True])
def test_deeper_model_checkpoints_reload_bit_for_bit(tmp_path, tf_format):
    enc, dec = SHAPES["3x2"]
    a = make_mlp(tmp_path, None, enc, dec, tag="ckpt")
    x, _, eps = inputs(4)
    a.train_step(x, x, eps)
    a.step_idx = 3
    a.save(tf_format=tf_format)
    assert "decoder/dense_2/kernel" in a._names and "encoder/dense_2/bias" in a._names
    b = make_mlp(tmp_path, None, enc, dec, tag="ckpt")
    b.set_weights({k: np.zeros_like(v) for k, v in b.get_weights().items()})
    assert b.load_latest_checkpoint() is True and b.get_step_idx() == 3
    assert bool((b.params == a.params).all()) and bool((b.adam_m == a.adam_m).all()) and bool((b.adam_v == a.adam_v).all())
    assert bool((b.adam_powers == a.adam_powers).all())
    assert np.array_equal(b.encode(x[:2]), a.encode(x[:2]))


def _episode(tmp_path, lib, mode, fused):
    from carla_ppo_b200 import _lib
    from carla_ppo_b200.actor import FusedActor
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.vae_common import create_encode_state_fn
    with math_mode(lib, mode):
        rgb, _ = committed_frames()
        env = ReplayEnv(rgb, episode_length=20, seed=3)
        enc, dec = SHAPES["3x2"]
        vae = make_mlp(tmp_path, mlp_weights(2, encoder_sizes=enc, decoder_sizes=dec), enc, dec, tag="actor", training=False)
        model = PPO((67,), env.action_space, initial_std=0.4, model_dir=str(tmp_path / ("agent%d" % fused)), seed=0)
        model.init_session(init_logging=False)
        if fused:
            actor = FusedActor(vae, model, MEAS)
            env.encode_state_fn, predict = actor.encode_state_fn, actor.predict
        else:
            env.encode_state_fn, predict = create_encode_state_fn(vae, MEAS), model.predict
        states, actions, rewards = [env.reset()], [], []
        terminal = False
        while not terminal:
            a, _ = predict(states[-1])
            s, r, terminal, _ = env.step(a)
            states.append(s); actions.append(np.array(a)); rewards.append(r)
        return states, actions, rewards


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2])
def test_fused_actor_takes_an_mlp_vae_and_reproduces_the_unfused_loop(tmp_path, lib, mode):
    fs, fa, fr = _episode(tmp_path, lib, mode, True)
    us, ua, ur = _episode(tmp_path, lib, mode, False)
    assert len(fs) == len(us) > 2
    assert all(np.array_equal(a, b) for a, b in zip(fs, us))
    assert all(np.array_equal(a, b) for a, b in zip(fa, ua))
    assert fr == ur


@pytest.mark.gpu
def test_train_runs_an_mlp_vae_on_the_default_fused_path(tmp_path):
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    rgb, _ = committed_frames()
    enc, dec = SHAPES["3x2"]
    params = dict(learning_rate=1e-4, lr_decay=1.0, discount_factor=0.99, gae_lambda=0.95, ppo_epsilon=0.2, initial_std=0.4,
                  value_scale=1.0, entropy_scale=0.01, horizon=16, num_epochs=2, num_episodes=2, batch_size=8,
                  vae_model="unused", vae_model_type=None, vae_z_dim=None, synchronous=True, fps=30, action_smoothing=0.0,
                  model_name="mlp_fused", reward_fn="reward_speed_centering_angle_multiply", seed=0, eval_interval=1,
                  record_eval=False, logging=False)
    vae = make_mlp(tmp_path, mlp_weights(2, encoder_sizes=enc, decoder_sizes=dec), enc, dec, tag="train", training=False)
    env = ReplayEnv(rgb, episode_length=24, seed=0)
    model = train(params, restart=False, env=env, vae=vae, models_root=str(tmp_path / "models"), interactive=False)
    assert params["vae_model_type"] == "mlp"
    assert model.get_episode_idx() == 2 and model.get_train_step_idx() > 0 and env.step_count > 0
    assert all(np.isfinite(v).all() for v in model.get_weights().values())


@pytest.mark.gpu
def test_loss_grad_repeats_bit_for_bit_and_mode_1_is_untouched(tmp_path, lib):
    """Two mode-2 loss_grad calls are bit-identical.  Mode 1, mode 2, mode 1 on the same inputs: the two mode-1 results
    and launch counts are identical, and mode 2 computed something else."""
    import torch
    from carla_ppo_b200 import _lib
    vae = make_mlp(tmp_path, mlp_weights())
    x, _, eps = inputs(8)
    xd, ed = dev(vae, x), dev(vae, eps)
    runs = []
    for mode in (_lib.MATH_3XTF32, _lib.MATH_TF32, _lib.MATH_TF32, _lib.MATH_3XTF32):
        with math_mode(lib, mode):
            vae._workspace(8, _lib.WS_TRAIN)                # size the workspace outside the counted call
            torch.cuda.synchronize()
            lib.cpb_reset_launch_count()
            vae.loss_grad_device(xd, xd, ed)
            torch.cuda.synchronize()
            runs.append((vae.grads.clone(), vae._losses.clone(), lib.cpb_launch_count()))
    assert torch.equal(runs[1][0], runs[2][0]) and torch.equal(runs[1][1], runs[2][1])
    assert torch.equal(runs[0][0], runs[3][0]) and torch.equal(runs[0][1], runs[3][1]) and runs[0][2] == runs[3][2]
    assert not torch.equal(runs[0][0], runs[1][0])


@pytest.mark.gpu
def test_a_mode_1_workspace_is_refused_in_mode_2(tmp_path, lib):
    import torch
    from carla_ppo_b200 import _lib
    vae = make_mlp(tmp_path, mlp_weights())
    x, _, eps = inputs(4)
    xd, ed = dev(vae, x), dev(vae, eps)
    cfg = vae._mlp_config(4)
    with math_mode(lib, _lib.MATH_3XTF32):
        need1 = lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), _lib.WS_TRAIN)
    with math_mode(lib, _lib.MATH_TF32):
        need2 = lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), _lib.WS_TRAIN)
        assert need2 > need1 > 0
        ws = torch.empty(need1, dtype=torch.uint8, device="cuda")
        grads = torch.empty_like(vae.grads)
        losses = torch.empty(2, device="cuda")
        torch.cuda.synchronize()
        before = lib.cpb_launch_count()
        st = lib.cpb_mlpvae_loss_grad(C.byref(cfg), vae.params.data_ptr(), xd.data_ptr(), xd.data_ptr(), ed.data_ptr(),
                                      grads.data_ptr(), losses.data_ptr(), None, ws.data_ptr(), need1,
                                      _lib.current_stream_handle())
        assert st == -3 and b"workspace too small" in lib.cpb_last_error()
        assert lib.cpb_launch_count() == before


@pytest.mark.gpu
def test_train_vae_cli_trains_the_mlp_vae_in_tf32(tmp_path):
    from PIL import Image
    from carla_ppo_b200.vae import train_vae
    rgb, _ = committed_frames()
    data = tmp_path / "data"
    (data / "rgb").mkdir(parents=True)
    for i in range(24):
        Image.fromarray(rgb[i]).save(data / "rgb" / ("%d.png" % i))
    vae = train_vae.main(["--dataset", str(data), "--batch_size", "8", "--max_epochs", "1", "--model_type", "mlp",
                          "--math_mode", "tf32", "--models_root", str(tmp_path / "models"), "-restart"])
    assert type(vae).__name__ == "MlpVAE" and "_mlp_zdim64_" in vae.model_dir
    assert vae.get_step_idx() >= 1
    assert np.isfinite(vae.evaluate(rgb[:8], rgb[:8], 8)).all()
    assert any(f.endswith(".npz") for f in os.listdir(vae.checkpoint_dir))
