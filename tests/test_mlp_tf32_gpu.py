"""Math mode 2 on the MlpVAE: its five frame-wide products (encoder/dense forward and weight gradient, decoder/dense_2
forward, data gradient and weight gradient) as ONE TF32 wgmma pass with both operands rounded to nearest.  Pinned here:

  * on the device's own inputs, each product is the fp32-summed product of the rounded operands (unit bar 2e-6), at a
    batch where the reductions over a frame run unsplit tiles and at B = 512 where they run k-split;
  * the whole model is within max(1e-5, 2 x err_tf32) of float64, err_tf32 being the distance of the TF32
    restatement (tests/mlp_tf32_oracle.py) from float64 on the same inputs;
  * results do not depend on the batch a frame is in, repeat bit for bit, and leave mode 1 bit-identical;
  * a workspace sized in mode 1 is refused in mode 2 before anything is launched.
Every test restores mode 1 when it ends."""
import ctypes as C
import os

import numpy as np
import pytest

import mlp_tf32_oracle
from helpers import committed_frames, rel_l2
from tf32_oracle import round_tf32

UNIT_TOL = 2e-6
FWD_TOL = 1e-5
IN = 38400
BUFFERS = ["x", "h1", "h2", "heads", "z", "g1", "g2", "logits", "ga", "gb"]


@pytest.fixture(scope="module")
def lib():
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(autouse=True)
def tf32_mode(lib):
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_TF32))
    yield
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_3XTF32))


def mlp_weights(seed=1, **kw):
    from oracle import vae_oracle as vo
    w = vo.mlp_glorot_init(seed, **kw)
    for k in w:                                   # non-zero biases: keep the ReLU pre-activations away from the kink
        if k.endswith("bias"):
            w[k] = (0.05 * np.random.RandomState(len(k)).randn(*w[k].shape)).astype(np.float32)
    return w


def make_mlp(tmp_path, w, loss="bce", z=64, ct=3, enc=(512, 256), dec=(256, 512)):
    from carla_ppo_b200.vae.models import MlpVAE
    vae = MlpVAE(source_shape=(80, 160, 3), target_shape=(80, 160, ct), z_dim=z, loss_fn=loss, encoder_sizes=enc,
                 decoder_sizes=dec, model_dir=str(tmp_path / ("mlp_zdim%d" % z)), seed=0)
    vae.init_session(init_logging=False)
    vae.set_weights(w)
    return vae


def inputs(n, z=64, seed=0):
    x = np.random.RandomState(seed).rand(n, 80, 160, 3).astype(np.float32)
    eps = np.random.RandomState(seed + 1).randn(n, z).astype(np.float32)
    return x, eps


def dev(vae, a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device=vae._device)


def read_ws(vae, batch, ws_mode, widths):
    """Named buffers of the last call that used workspace `ws_mode`, read back from the device as [batch, width]."""
    import torch
    from carla_ppo_b200 import _lib
    offs = (C.c_int64 * len(BUFFERS))()
    cfg = vae._mlp_config(batch)
    assert _lib.load().cpb_debug_mlpvae_buffer_offsets(C.byref(cfg), ws_mode, offs, len(BUFFERS)) == len(BUFFERS)
    ws = vae._ws[ws_mode]
    out = {}
    for nm, width in widths.items():
        o = offs[BUFFERS.index(nm)]
        out[nm] = ws[o:o + 4 * batch * width].view(torch.float32).cpu().numpy().astype(np.float64).reshape(batch, width)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [6, 512])
def test_frame_wide_products_on_the_devices_own_inputs(tmp_path, batch):
    """Forward: h1 = relu(r(x) r(W_enc) + b) and logits = r(g2) r(W_dec2) + b on the device's own x and g2.  Backward:
    both weight gradients against r(in)^T r(g) on the device's own operands; the data gradient of decoder/dense_2
    (g(g2) = (r(dlogits) r(W_dec2)^T) * (g2 > 0), overwritten later in the step) through the gradient of
    decoder/dense_1, g1^T g(g2), which the fp32 SIMT kernels compute from it."""
    from carla_ppo_b200 import _lib
    r = round_tf32
    w = mlp_weights()
    vae = make_mlp(tmp_path, w)
    x, eps = inputs(batch)
    vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps))
    t = read_ws(vae, batch, _lib.WS_FORWARD, {"x": IN, "h1": 512, "g2": 512, "logits": IN})
    assert np.array_equal(t["x"], x.reshape(batch, -1))
    err = rel_l2(t["h1"], np.maximum(r(t["x"]) @ r(w["encoder/dense/kernel"]) + w["encoder/dense/bias"], 0.0))
    assert err < UNIT_TOL, ("encoder/dense fwd", err)
    err = rel_l2(t["logits"], r(t["g2"]) @ r(w["decoder/dense_2/kernel"]) + w["decoder/dense_2/bias"])
    assert err < UNIT_TOL, ("decoder/dense_2 fwd", err)

    vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
    got = vae.get_grads()
    t = read_ws(vae, batch, _lib.WS_TRAIN, {"x": IN, "g1": 256, "g2": 512, "logits": IN, "gb": 512})
    dlog = t["logits"]                             # d loss / d logits after loss_grad
    err = rel_l2(got["encoder/dense/kernel"], r(t["x"]).T @ r(t["gb"]))
    assert err < UNIT_TOL, ("encoder/dense wgrad", err)
    err = rel_l2(got["decoder/dense_2/kernel"], r(t["g2"]).T @ r(dlog))
    assert err < UNIT_TOL, ("decoder/dense_2 wgrad", err)
    g_g2 = (r(dlog) @ r(w["decoder/dense_2/kernel"]).T) * (t["g2"] > 0)
    err = rel_l2(got["decoder/dense_1/kernel"], t["g1"].T @ g_g2)
    assert err < UNIT_TOL, ("decoder/dense_2 dgrad", err)


CASES = {   # z, target channels, loss, encoder sizes, decoder sizes
    "z64_bce_rgb": (64, 3, "bce", (512, 256), (256, 512)),
    "z32_bce_rgb": (32, 3, "bce", (512, 256), (256, 512)),
    "z64_mse_seg": (64, 1, "mse", (512, 256), (256, 512)),
    # enc1 = 96: 32-wide tensor-core tiles on a width that is not a multiple of 64; dec2 = 64: the weight gradient
    # with fewer than 128 rows (run as its transpose)
    "odd_widths": (64, 3, "bce", (96, 64), (160, 64)),
}


def _gate(t32, ref):
    return max(FWD_TOL, 2.0 * rel_l2(t32, ref))


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_model_matches_float64_within_twice_the_tf32_restatement(tmp_path, case):
    """6 random frames.  Forward tensors, losses and all 14 gradients against plain float64, gated at
    max(1e-5, 2 x err_tf32) (gradients: both restatements on the device's ReLU activity pattern); then two Adam steps,
    gated by the restatement's own two steps.  The device is closer to the TF32 restatement than to float64 for mean."""
    from carla_ppo_b200 import _lib
    from oracle import vae_oracle as vo
    z, ct, loss, enc, dec = CASES[case]
    w = mlp_weights(1, target_channels=ct, z_dim=z, encoder_sizes=enc, decoder_sizes=dec)
    vae = make_mlp(tmp_path, w, loss, z, ct, enc, dec)
    x, eps = inputs(6, z)
    y = x if ct == 3 else np.random.RandomState(9).rand(6, 80, 160, 1).astype(np.float32)
    out = vae.forward_device(dev(vae, x), dev(vae, y), dev(vae, eps), want_reconstruction=True, want_latents=True)
    fwd = {k: out[k].cpu().numpy().astype(np.float64) for k in ("mean", "logvar", "z", "reconstruction")}
    vae.loss_grad_device(dev(vae, x), dev(vae, y), dev(vae, eps))
    got = vae.get_grads()
    losses = vae._losses.cpu().numpy().astype(np.float64)
    t = read_ws(vae, 6, _lib.WS_TRAIN, {"h1": enc[0], "h2": enc[1], "g1": dec[0], "g2": dec[1]})
    masks = {k: v > 0 for k, v in t.items()}
    ref = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, loss, tc_round=lambda a: a, relu_masks=masks)
    t32 = mlp_tf32_oracle.loss_and_grads(w, x, y, eps, loss, relu_masks=masks)
    for k in ("mean", "logvar", "z"):
        gate = _gate(t32[k], ref[k])
        assert rel_l2(fwd[k], ref[k]) < gate, (k, rel_l2(fwd[k], ref[k]), gate)
    rec_ref = vo.sigmoid(ref["logits"])
    gate = _gate(vo.sigmoid(t32["logits"]), rec_ref)
    assert rel_l2(fwd["reconstruction"], rec_ref) < gate
    for i, k in enumerate(("recon", "kl")):
        scale = max(abs(ref[k]), 1.0)
        gate = max(FWD_TOL, 2.0 * abs(t32[k] - ref[k]) / scale)
        assert abs(losses[i] - ref[k]) / scale < gate, (k, losses[i], ref[k], t32[k])
    assert len(ref["grads"]) == 14
    for name, g in ref["grads"].items():
        gate = _gate(t32["grads"][name], g)
        assert rel_l2(got[name], g) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], g), gate)
    assert rel_l2(fwd["mean"], t32["mean"]) < rel_l2(fwd["mean"], ref["mean"])
    # two Adam steps from the same weights: device vs float64, gated by the restatement's own distance from float64
    p64 = {k: v.astype(np.float64) for k, v in w.items()}
    p32 = {k: v.astype(np.float64) for k, v in w.items()}
    st64, st32 = vo.adam_init_state(p64), vo.adam_init_state(p32)
    for _ in range(2):
        vae.train_step(x, y, eps)
        vo.mlp_train_step(p64, st64, x, y, eps, lr=1e-4, loss_type=loss)
        vo.adam_apply(p32, mlp_tf32_oracle.loss_and_grads(p32, x, y, eps, loss)["grads"], st32, 1e-4)
    gotw = vae.get_weights()
    for name in p64:
        gate = _gate(p32[name], p64[name])
        assert rel_l2(gotw[name], p64[name]) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(gotw[name], p64[name]), gate)


@pytest.mark.gpu
def test_encoding_does_not_depend_on_the_batch(tmp_path):
    """The k-split and every tile choice are fixed by the layer shapes: 8 frames encode bit for bit as their quarters."""
    w = mlp_weights()
    vae = make_mlp(tmp_path, w)
    x, _ = inputs(8)
    whole, whole_lv = vae.encode_device(dev(vae, x), return_logvar=True)
    parts = [vae.encode_device(dev(vae, x[i:i + 2]), return_logvar=True) for i in range(0, 8, 2)]
    import torch
    assert torch.equal(whole, torch.cat([p[0] for p in parts])) and torch.equal(whole_lv, torch.cat([p[1] for p in parts]))


@pytest.mark.gpu
def test_loss_grad_repeats_bit_for_bit_and_mode_1_is_untouched(tmp_path, lib):
    """Two mode-2 loss_grad calls are bit-identical.  Mode 1, mode 2, mode 1 on the same inputs: the two mode-1 results
    and launch counts are identical, and mode 2 computed something else."""
    import torch
    from carla_ppo_b200 import _lib
    vae = make_mlp(tmp_path, mlp_weights())
    x, eps = inputs(8)
    xd, ed = dev(vae, x), dev(vae, eps)
    runs = []
    for mode in (_lib.MATH_3XTF32, _lib.MATH_TF32, _lib.MATH_TF32, _lib.MATH_3XTF32):
        _lib.check(lib.cpb_set_math_mode(mode))
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
    x, eps = inputs(4)
    xd, ed = dev(vae, x), dev(vae, eps)
    cfg = vae._mlp_config(4)
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_3XTF32))
    need1 = lib.cpb_mlpvae_workspace_bytes(C.byref(cfg), _lib.WS_TRAIN)
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_TF32))
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
