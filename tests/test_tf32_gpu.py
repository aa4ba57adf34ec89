"""Math mode 2: the ConvVAE's tensor-core layers (conv2-4, deconv1-3: forward, data gradient, weight gradient) as ONE
TF32 wgmma pass with both operands rounded to the nearest TF32 value.  Not fp32-accurate by design; what is pinned:

  * the kernels compute exactly the products of the rounded operands, summed in fp32 (unit bar 2e-6, as for 3xTF32),
    and the rounding is to nearest, not the tensor core's truncation (no bias on all-positive data);
  * every interior layer, on the device's own inputs, matches relu(contract(round_tf32(in), round_tf32(W)) + b);
  * the whole model is within max(1e-5, 2 x err_tf32) of float64, err_tf32 being the distance of the "TF32
    restatement" (tests/tf32_oracle.py: the float64 oracle with round_tf32 applied to the same operands) from
    float64 on the same inputs;
  * switching modes leaves mode 1 bit-identical."""
import os
import subprocess
import sys

import numpy as np
import pytest

import tf32_oracle
from harness import conv_relu_masks, conv_workspace, dev, lib, library_state, make_conv_vae, math_mode  # noqa: F401
from helpers import committed_frames, kat, rel_l2, shipped_vae_weights
from tf32_oracle import round_tf32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNIT_TOL = 2e-6          # the tensor-core unit bar (tests/test_tc_gpu.py): only the fp32 accumulation differs
FWD_TOL = 1e-5


def test_math_mode_2_is_accepted_and_bad_modes_are_rejected(lib):
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_TF32))
    assert lib.cpb_get_math_mode() == _lib.MATH_TF32
    for bad in (3, -1):
        assert lib.cpb_set_math_mode(bad) == -1
        assert b"math mode must be" in lib.cpb_last_error()
        assert lib.cpb_get_math_mode() == _lib.MATH_TF32          # a rejected value leaves the mode as it was
    for mode in (_lib.MATH_SIMT, _lib.MATH_3XTF32, _lib.MATH_TF32):
        _lib.check(lib.cpb_set_math_mode(mode))
        assert lib.cpb_get_math_mode() == mode


def test_train_vae_cli_has_the_math_mode_flag():
    from carla_ppo_b200.vae import train_vae
    p = train_vae.build_parser()
    assert p.parse_args([]).math_mode == "3xtf32"
    assert train_vae.MATH_MODES[p.parse_args(["--math_mode", "tf32"]).math_mode] == 2
    with pytest.raises(SystemExit):
        p.parse_args(["--math_mode", "fp16"])


def test_tf32_restatement_rounds_exactly_the_tensor_core_contractions():
    """The restatement rounds the 18 contractions of conv2-4 / deconv1-3 in a full forward + backward (forward, data
    gradient, weight gradient each) and none of the 5 of conv1 / deconv4; with an identity rounding it is the oracle
    bit for bit, and the oracle's primitives are restored afterwards."""
    from oracle import vae_oracle as vo
    w = vo.glorot_init(0, target_channels=1)
    x = np.random.RandomState(0).rand(2, 80, 160, 3).astype(np.float32)
    y = np.random.RandomState(4).rand(2, 80, 160, 1).astype(np.float32)
    eps = np.random.RandomState(1).randn(2, 64).astype(np.float32)
    ref = vo.loss_and_grads(w, x, y, eps, "bce")
    with tf32_oracle.rounded_tensor_core_contractions(lambda a: a) as calls:
        same = vo.loss_and_grads(w, x, y, eps, "bce")
    assert calls == {"rounded": 18, "plain": 5}
    assert all(np.array_equal(same["grads"][k], ref["grads"][k]) for k in ref["grads"]) and same["recon"] == ref["recon"]
    assert vo.conv_gather.__module__ == "oracle.vae_oracle" and vo.conv_wgrad.__module__ == "oracle.vae_oracle"
    t32 = tf32_oracle.loss_and_grads(w, x, y, eps, "bce")
    assert not np.array_equal(t32["mean"], ref["mean"])
    x0 = np.float32([1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, -1.0 - 2 ** -11])    # ties go away from zero
    assert np.array_equal(round_tf32(x0), [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -1.0 - 2 ** -10])


# ----------------------------------------------------------------------------- kernel units
def _gemm(lib, a, bt):
    import torch
    from carla_ppo_b200 import _lib
    m, k = a.shape
    n = bt.shape[0]
    ta, tb = torch.tensor(a, device="cuda"), torch.tensor(bt, device="cuda")
    d = torch.full((m, n), float("nan"), device="cuda")
    scratch = torch.empty(2 * n * k, device="cuda")
    with math_mode(lib, _lib.MATH_TF32):
        _lib.check(lib.cpb_debug_tc_gemm(ta.data_ptr(), tb.data_ptr(), d.data_ptr(), m, n, k, scratch.data_ptr(),
                                         _lib.current_stream_handle()))
        torch.cuda.synchronize()
    return d.cpu().numpy()


def _wgrad(lib, big, small):
    import torch
    from carla_ppo_b200 import _lib
    m, i = big.shape
    j = small.shape[1]
    tb, ts = torch.tensor(big, device="cuda"), torch.tensor(small, device="cuda")
    out = torch.full((i, j), float("nan"), device="cuda")
    part = torch.zeros(2 * i * j, device="cuda")          # the debug entry uses 2 splits
    with math_mode(lib, _lib.MATH_TF32):
        _lib.check(lib.cpb_debug_tc_wgrad(tb.data_ptr(), ts.data_ptr(), out.data_ptr(), m, i, j, 0, part.data_ptr(),
                                          _lib.current_stream_handle()))
        torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k", [(128, 32, 32), (300, 32, 576), (1, 64, 64), (257, 64, 800), (4096, 128, 256),
                                   (20000, 128, 96), (513, 256, 2048), (130, 512, 128)])
def test_tf32_gemm_is_the_product_of_rounded_operands(lib, m, n, k):
    rs = np.random.RandomState(m + n + k)
    a = rs.randn(m, k).astype(np.float32)
    bt = rs.randn(n, k).astype(np.float32)
    got = _gemm(lib, a, bt)
    assert np.isfinite(got).all()
    assert rel_l2(got, round_tf32(a) @ round_tf32(bt).T) < UNIT_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("m,i,j", [(4096, 128, 128), (5000, 256, 64), (4100, 128, 32), (1031, 384, 256),
                                   (32, 128, 32), (33, 128, 64), (95, 256, 32), (127, 200, 64), (2048, 640, 32),
                                   (3001, 1024, 64), (16384, 128, 64), (777, 136, 96)])
def test_tf32_wgrad_is_the_product_of_rounded_operands(lib, m, i, j):
    rs = np.random.RandomState(m + i + j)
    big = rs.randn(m, i).astype(np.float32)
    small = rs.randn(m, j).astype(np.float32)
    got = _wgrad(lib, big, small)
    assert rel_l2(got, round_tf32(big).T @ round_tf32(small)) < UNIT_TOL


@pytest.mark.gpu
def test_tf32_rounds_to_nearest_not_toward_zero(lib):
    """All-positive operands at K = 4096: rounding to nearest leaves the mean signed relative error against exact
    float64 at ~1e-6 (the rounding errors have no sign); the tensor core's own truncation of both operands would
    make it ~-6.5e-4 (every product too small), 30x beyond the 2e-5 bar."""
    rs = np.random.RandomState(7)
    a = rs.rand(256, 4096).astype(np.float32)
    bt = rs.rand(128, 4096).astype(np.float32)
    got = _gemm(lib, a, bt)
    exact = a.astype(np.float64) @ bt.astype(np.float64).T
    assert rel_l2(got, round_tf32(a) @ round_tf32(bt).T) < UNIT_TOL
    assert abs(np.mean((got - exact) / exact)) < 2e-5
    got = _wgrad(lib, a.T.copy(), bt.T.copy())                # the same contraction through the weight-gradient kernel
    assert rel_l2(got, round_tf32(a) @ round_tf32(bt).T) < UNIT_TOL
    assert abs(np.mean((got - exact) / exact)) < 2e-5


_SNIPPET = r"""
import sys, hashlib, numpy as np, torch
sys.path.insert(0, %r)
sys.path.insert(0, %r)
from carla_ppo_b200 import _lib
from tf32_oracle import round_tf32
lib = _lib.load()
_lib.check(lib.cpb_set_math_mode(_lib.MATH_TF32))
rs = np.random.RandomState(3)
m, n, k = 3000, 128, 288
a = rs.randn(m, k).astype(np.float32); bt = rs.randn(n, k).astype(np.float32)
ta, tb = torch.tensor(a, device="cuda"), torch.tensor(bt, device="cuda")
d = torch.empty(m, n, device="cuda"); sc = torch.empty(2 * n * k, device="cuda")
_lib.check(lib.cpb_debug_tc_gemm(ta.data_ptr(), tb.data_ptr(), d.data_ptr(), m, n, k, sc.data_ptr(), _lib.current_stream_handle()))
torch.cuda.synchronize()
print("HASH", hashlib.sha256(d.cpu().numpy().tobytes()).hexdigest())
ref = round_tf32(a) @ round_tf32(bt).T
print("ERR", float(np.linalg.norm(d.cpu().numpy() - ref) / np.linalg.norm(ref)))
"""


@pytest.mark.gpu
def test_tf32_gemm_is_bit_identical_across_cluster_sizes():
    """CPB_TC_CLUSTER only changes who copies which slice of the (hi-only) weight tile, never the arithmetic."""
    hashes, errs = {}, {}
    for cs in ("1", "2", "4"):
        env = dict(os.environ, CPB_TC_CLUSTER=cs)
        res = subprocess.run([sys.executable, "-c", _SNIPPET % (ROOT, os.path.join(ROOT, "tests"))], env=env,
                             capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stderr[-2000:]
        hashes[cs] = [ln for ln in res.stdout.splitlines() if ln.startswith("HASH")][0]
        errs[cs] = float([ln for ln in res.stdout.splitlines() if ln.startswith("ERR")][0].split()[1])
    assert hashes["1"] == hashes["2"] == hashes["4"]
    assert errs["1"] < UNIT_TOL, errs


# ----------------------------------------------------------------------------- model level
def config1_inputs(n=32):
    x = np.random.RandomState(0).rand(n, 80, 160, 3).astype(np.float32)
    eps = np.random.RandomState(1).randn(n, 64).astype(np.float32)
    return x, eps


@pytest.mark.gpu
def test_every_tensor_core_layer_on_the_devices_own_inputs(tmp_path, lib):
    """One forward at B = 32; each interior layer's output against relu(contract(round_tf32(in), round_tf32(W)) + b)
    in float64 on the input the DEVICE computed, so no error of an earlier layer is carried into the comparison."""
    from carla_ppo_b200 import _lib
    from oracle import vae_oracle as vo
    w = shipped_vae_weights()[0]
    vae = make_conv_vae(tmp_path, w)
    x, eps = config1_inputs(32)
    with math_mode(lib, _lib.MATH_TF32):
        vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps))
    t = {k: v.cpu().numpy().astype(np.float64) for k, v in conv_workspace(vae, 32, _lib.WS_FORWARD).items() if k != "g"}
    r = round_tf32
    layers = [("encoder/conv2", vo.conv_gather, "a1", "a2"), ("encoder/conv3", vo.conv_gather, "a2", "a3"),
              ("encoder/conv4", vo.conv_gather, "a3", "a4"), ("decoder/deconv1", vo.conv_scatter, "d1", "b1"),
              ("decoder/deconv2", vo.conv_scatter, "b1", "b2"), ("decoder/deconv3", vo.conv_scatter, "b2", "b3")]
    for name, contract, src, dst in layers:
        ref = np.maximum(contract(r(t[src]), r(w[name + "/kernel"])) + w[name + "/bias"], 0.0)
        err = rel_l2(t[dst], ref)
        assert err < UNIT_TOL, "%s: %.3e" % (name, err)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["mse", "bce"])
@pytest.mark.parametrize("which", ["shipped", "glorot0"])
def test_model_matches_float64_within_twice_the_tf32_restatement(tmp_path, lib, which, loss):
    """BASELINE config 1 (32 random frames).  Forward tensors, losses and all 22 gradients against plain float64, gated
    at max(1e-5, 2 x err_tf32), err_tf32 = the TF32 restatement's own distance from float64 (gradients: both oracle
    runs on the device's ReLU activity pattern, as tests/vae_checks.py::grad_check).  Plus: the device is closer
    to the TF32 restatement than to float64 for `mean`, and for each loss whose TF32 shift from float64 stands above
    the float32 rounding level (2 x the distance of the float32 CPU restatement from float64) -- below that level
    the comparison would measure float32 rounding, not the single pass."""
    import torch
    from carla_ppo_b200 import _lib
    from oracle import torch_ref
    from oracle import vae_oracle as vo
    w = shipped_vae_weights()[0] if which == "shipped" else vo.glorot_init(0)
    vae = make_conv_vae(tmp_path, w, loss=loss)
    x, eps = config1_inputs(32)
    with math_mode(lib, _lib.MATH_TF32):
        out = vae.forward_device(dev(vae, x), dev(vae, x), dev(vae, eps), want_reconstruction=True, want_latents=True)
        fwd = {k: out[k].cpu().numpy().astype(np.float64) for k in ("mean", "logvar", "z", "reconstruction")}
        vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
        got = vae.get_grads()
        losses = vae._losses.cpu().numpy().astype(np.float64)
    masks = conv_relu_masks(vae, 32)
    ref = vo.loss_and_grads(w, x, x, eps, loss, relu_masks=masks)
    t32 = tf32_oracle.loss_and_grads(w, x, x, eps, loss, relu_masks=masks)
    for k in ("mean", "logvar", "z"):
        gate = max(FWD_TOL, 2.0 * rel_l2(t32[k], ref[k]))
        assert rel_l2(fwd[k], ref[k]) < gate, (k, rel_l2(fwd[k], ref[k]), gate)
    rec_ref = vo.sigmoid(ref["logits"]).reshape(32, -1)
    gate = max(FWD_TOL, 2.0 * rel_l2(vo.sigmoid(t32["logits"]).reshape(32, -1), rec_ref))
    assert rel_l2(fwd["reconstruction"], rec_ref) < gate
    for i, k in enumerate(("recon", "kl")):
        # glorot0's KL (~0.05) is a cancelling sum: absolute errors there, as in tests/test_vae_gpu.py
        scale = 1.0 if (which == "glorot0" and k == "kl") else abs(ref[k])
        gate = max(FWD_TOL, 2.0 * abs(t32[k] - ref[k]) / scale)
        assert abs(losses[i] - ref[k]) / scale < gate, (k, losses[i], ref[k], t32[k])
    for name, g in ref["grads"].items():
        gate = max(FWD_TOL, 2.0 * rel_l2(t32["grads"][name], g))
        assert rel_l2(got[name], g) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], g), gate)
    # the single pass ran, with rounding to nearest
    assert rel_l2(fwd["mean"], t32["mean"]) < rel_l2(fwd["mean"], ref["mean"])
    r32 = torch_ref.vae_loss_and_grads(w, x, x, eps, loss, dtype=torch.float32)
    for i, k in enumerate(("recon", "kl")):
        if abs(t32[k] - ref[k]) > 2.0 * abs(r32[k] - ref[k]):
            assert abs(losses[i] - t32[k]) < abs(losses[i] - ref[k]), (k, losses[i], t32[k], ref[k])


@pytest.mark.gpu
def test_known_answer_shipped_checkpoint_in_tf32(tmp_path, lib):
    """KAT-1 in mode 2: shipped rgb checkpoint-232 on the 128 committed frames stays within the reference-held bars of
    tests/test_vae_gpu.py::test_known_answer_shipped_checkpoint_on_shipped_frames: 1 % (reconstruction) and 5 % (KL)
    of the reference's own logged validation losses."""
    from carla_ppo_b200 import _lib
    w = shipped_vae_weights()[0]
    rgb, _ = committed_frames()
    vae = make_conv_vae(tmp_path, w, loss="bce")
    eps = np.random.RandomState(7).randn(rgb.shape[0], 64).astype(np.float32)
    with math_mode(lib, _lib.MATH_TF32):
        losses = vae.forward_device(dev(vae, rgb), dev(vae, rgb), dev(vae, eps))["losses"].cpu().numpy()
    k = kat()
    logged = np.mean([v for _, v in k["logged"]["val"]["vae/reconstruction_loss"]])
    logged_kl = np.mean([v for _, v in k["logged"]["val"]["vae/kl_loss"]])
    assert abs(losses[0] - logged) / logged < 0.01
    assert abs(losses[1] - logged_kl) / logged_kl < 0.05


@pytest.mark.gpu
def test_mode_1_is_untouched_by_mode_2(tmp_path, lib):
    """loss_grad in mode 1, then mode 2, then mode 1 on the same inputs: the two mode-1 results are bit-identical (the
    weight images are rebuilt for the mode of each call), and mode 2 computed something else."""
    import torch
    from carla_ppo_b200 import _lib
    from oracle import vae_oracle as vo
    vae = make_conv_vae(tmp_path, vo.glorot_init(0))
    x, eps = config1_inputs(8)
    res = []
    for mode in (_lib.MATH_3XTF32, _lib.MATH_TF32, _lib.MATH_3XTF32):
        with math_mode(lib, mode):
            vae.loss_grad_device(dev(vae, x), dev(vae, x), dev(vae, eps))
            res.append((vae.grads.clone(), vae._losses.clone()))
    assert torch.equal(res[0][0], res[2][0]) and torch.equal(res[0][1], res[2][1])
    assert not torch.equal(res[0][0], res[1][0])
