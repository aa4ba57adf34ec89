"""Checks that several GPU test modules share: the ConvVAE's gradients against the float64 oracle and the weights that
keep its ReLU pre-activations off the kink, and the MlpVAE's frame-wide products on the device's own operands."""
import numpy as np

import mlp_depth_oracle as mdo
from harness import conv_relu_masks, dev, mlp_workspace
from helpers import rel_l2
from tf32_oracle import round_tf32

FWD_TOL = 1e-5
UNIT_TOL = 2e-6          # the tensor-core unit bar: only the fp32 accumulation differs
IN = 38400               # the MlpVAE's input width, 80 x 160 x 3


# ------------------------------------------------------------------------------------------------------ ConvVAE
def grad_check(vae, oracle, w, x, y, eps, loss, beta=1.0, kl_tolerance=0.0, floor=2e-5):
    """Gradients vs the float64 oracle evaluated on the DEVICE's ReLU activity pattern (see
    oracle.loss_and_grads: a sign flip of a ~0 pre-activation is not an arithmetic error), plus the check that
    the device pattern differs from float64's only on a vanishing fraction of elements whose float64
    pre-activation is negligible."""
    from oracle import torch_ref
    import torch
    vae.loss_grad_device(dev(vae, x), dev(vae, y), dev(vae, eps))
    got = vae.get_grads()
    losses = vae._losses.cpu().numpy()
    masks = conv_relu_masks(vae, x.shape[0])
    xs = x.astype(np.float32) / 255.0 if x.dtype == np.uint8 else x
    ys = xs if y is x else y
    ref = oracle.loss_and_grads(w, xs, ys, eps, loss, beta, kl_tolerance, relu_masks=masks)
    ref32 = torch_ref.vae_loss_and_grads(w, xs, ys, eps, loss, beta, kl_tolerance, dtype=torch.float32)
    assert abs(losses[0] - ref["recon"]) / ref["recon"] < FWD_TOL
    for name, pre in ref["relu_pre"].items():
        flips = masks[name] != (pre > 0)
        assert flips.mean() < 1e-4, (name, flips.mean())
        if flips.any():
            assert np.abs(pre[flips]).max() < 2e-5 * np.sqrt(np.mean(pre * pre)), (name, np.abs(pre[flips]).max())
    worst = 0.0
    for name, g in ref["grads"].items():
        err = rel_l2(got[name], g)
        cpu32 = rel_l2(ref32["grads"][name], g)
        tol = max(2.0 * cpu32, floor)
        assert err < tol, "%s: rel err %.3e (fp32 CPU restatement: %.3e)" % (name, err, cpu32)
        worst = max(worst, err)
    return worst


def shift_away_from_zero(oracle, w, x, eps, margin=5e-5):
    """Returns weights whose ReLU pre-activations on (x, eps) are ALL at least `margin` away from zero: each bias is
    moved (per output channel, layer by layer) by the smallest shift that empties the band (-margin, margin)."""
    w = {k: v.copy() for k, v in w.items()}
    order = [("encoder/conv%d" % i, "conv%d" % i) for i in range(1, 5)] + [("decoder/deconv%d" % i, "deconv%d" % i) for i in range(1, 4)]
    for tf_name, key in order:
        for _ in range(8):
            pre = oracle.loss_and_grads(w, x, x, eps, "mse", want_grads=False)["relu_pre"][key]
            flat = pre.reshape(-1, pre.shape[-1])
            if np.abs(flat).min() >= margin:
                break
            b = w[tf_name + "/bias"].astype(np.float64)
            for c in range(flat.shape[1]):
                col = np.sort(flat[:, c])
                # candidate shifts: move the column so that the band falls into the widest gap near zero
                inside = col[(col > -64 * margin) & (col < 64 * margin)]
                if inside.size == 0 or np.abs(col).min() >= margin:
                    continue
                pts = np.concatenate([[-64 * margin], inside, [64 * margin]])
                gaps = np.diff(pts)
                j = int(np.argmax(gaps))
                if gaps[j] < 2.2 * margin:
                    continue
                b[c] -= 0.5 * (pts[j] + pts[j + 1])        # centre of the widest gap goes to zero
            w[tf_name + "/bias"] = b.astype(np.float32)
    return w


# ------------------------------------------------------------------------------------------------------ MlpVAE
def mlp_weights(seed=1, **kw):
    w = mdo.glorot_init(seed, **kw)
    for k in w:                                   # non-zero biases: keep the ReLU pre-activations away from the kink
        if k.endswith("bias"):
            w[k] = (0.05 * np.random.RandomState(len(k)).randn(*w[k].shape)).astype(np.float32)
    return w


def inputs(n, z=64, ct=3, seed=0):
    x = np.random.RandomState(seed).rand(n, 80, 160, 3).astype(np.float32)
    eps = np.random.RandomState(seed + 1).randn(n, z).astype(np.float32)
    y = x if ct == 3 else np.random.RandomState(seed + 9).rand(n, 80, 160, 1).astype(np.float32)
    return x, y, eps


def forward_products(vae, w, batch, frames=None):
    """After a mode-2 forward call: the first encoder layer's and the output layer's forward products on the device's
    own rows (`frames`, or all) against the fp32-summed product of the rounded operands -> {name: rel err}."""
    from carla_ppo_b200 import _lib
    r = round_tf32
    enc, dec = vae.encoder_sizes, vae.decoder_sizes
    out_name = "decoder/dense_%d" % len(dec)
    last = "g%d" % (len(dec) - 1)
    t = mlp_workspace(vae, batch, _lib.WS_FORWARD, {"x": IN, "h0": enc[0], last: dec[-1], "logits": IN}, frames)
    return {"first encoder layer fwd": rel_l2(t["h0"], np.maximum(r(t["x"]) @ r(w["encoder/dense/kernel"]) + w["encoder/dense/bias"], 0.0)),
            "output layer fwd": rel_l2(t["logits"], r(t[last]) @ r(w[out_name + "/kernel"]) + w[out_name + "/bias"])}


def backward_products(vae, w, batch, frames=None):
    """After a mode-2 loss_grad call: the first encoder layer's and the output layer's weight gradients, and the output
    layer's data gradient through the weight gradient of the last hidden decoder layer (which the fp32 SIMT kernels
    compute from it), against the same products over the rows `frames` (all of them when None; a batch whose other
    rows are exactly 0 otherwise) -> {name: rel err}."""
    from carla_ppo_b200 import _lib
    r = round_tf32
    enc, dec = vae.encoder_sizes, vae.decoder_sizes
    out_name = "decoder/dense_%d" % len(dec)
    last = "g%d" % (len(dec) - 1)
    got = vae.get_grads()
    below = "z" if len(dec) == 1 else "g%d" % (len(dec) - 2)
    t = mlp_workspace(vae, batch, _lib.WS_TRAIN, {"x": IN, below: 64 if len(dec) == 1 else dec[-2], last: dec[-1], "logits": IN,
                                            "gb": enc[0]}, frames)
    dlog = t["logits"]                             # d loss / d logits after loss_grad
    g_last = (r(dlog) @ r(w[out_name + "/kernel"]).T) * (t[last] > 0)
    return {"first encoder layer wgrad": rel_l2(got["encoder/dense/kernel"], r(t["x"]).T @ r(t["gb"])),
            "output layer wgrad": rel_l2(got[out_name + "/kernel"], r(t[last]).T @ r(dlog)),
            "output layer dgrad": rel_l2(got["decoder/dense_%d/kernel" % (len(dec) - 1) if len(dec) > 1 else "decoder/dense/kernel"],
                                         t[below].T @ g_last)}
