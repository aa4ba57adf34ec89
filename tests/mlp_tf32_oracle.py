"""The "TF32 restatement" of the MlpVAE oracle (test infrastructure for math mode 2 on the MlpVAE).

Math mode 2 runs the MlpVAE's five frame-wide products -- encoder/dense forward and weight gradient, decoder/dense_2
forward, data gradient and weight gradient -- on rounded operands (both rounded to the nearest TF32 value) and sums in
fp32; the other fifteen contractions of a forward + backward stay fp32.  The restatement is
oracle.vae_oracle.mlp_loss_and_grads with exactly those five products' operands rounded, everything else in float64.

The oracle writes its products as inline `@`, so they cannot be swapped from outside as the ConvVAE restatement
(tests/tf32_oracle.py) swaps its convolution primitives.  This module restates the oracle's arithmetic line for line,
with every contraction going through `mm`; with an identity rounding and no masks it is the oracle bit for bit
(tests/test_mlp_tf32_cpu.py pins that), so the copy cannot drift from the oracle unnoticed.

relu_masks (optional, {"h1", "h2", "g1", "g2"} -> bool arrays): the ReLU activity pattern to use instead of the sign
of the restatement's own pre-activations, as in vae_oracle.loss_and_grads -- a device run and a restatement then
differentiate the same piecewise-linear function."""
import numpy as np

from oracle import vae_oracle as vo
from tf32_oracle import round_tf32

TC_PRODUCTS = ("enc.fwd", "dec2.fwd", "dec2.dgrad", "enc.wgrad", "dec2.wgrad")


def loss_and_grads(params, x, y, eps, loss_type="mse", beta=1.0, kl_tolerance=0.0, tc_round=round_tf32, relu_masks=None,
                   calls=None):
    """vo.mlp_loss_and_grads (float64) with tc_round applied to both operands of the five frame-wide products.
    calls (optional dict) counts the rounded and the plain contractions."""
    dtype = np.float64
    if calls is not None:
        calls.setdefault("rounded", 0); calls.setdefault("plain", 0)

    def mm(name, a, b):
        hit = name in TC_PRODUCTS
        if calls is not None:
            calls["rounded" if hit else "plain"] += 1
        return tc_round(a) @ tc_round(b) if hit else a @ b

    def relu(pre, key):
        return np.maximum(pre, 0.0) if relu_masks is None else pre * relu_masks[key]

    def active(h, key):
        return (h > 0) if relu_masks is None else relu_masks[key]

    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    x = np.asarray(x, dtype); y = np.asarray(y, dtype); eps = np.asarray(eps, dtype)
    vo.verify_range(x); vo.verify_range(y)
    b = x.shape[0]
    xf = x.reshape(b, -1); yf = y.reshape(b, -1)
    h1 = relu(mm("enc.fwd", xf, p["encoder/dense/kernel"]) + p["encoder/dense/bias"], "h1")
    h2 = relu(mm("enc1.fwd", h1, p["encoder/dense_1/kernel"]) + p["encoder/dense_1/bias"], "h2")
    mean = mm("mean.fwd", h2, p["mean/kernel"]) + p["mean/bias"]
    logvar = mm("logvar.fwd", h2, p["logstd_sqare/kernel"]) + p["logstd_sqare/bias"]
    std = np.exp(0.5 * logvar)
    z = mean + eps * std
    g1 = relu(mm("dec.fwd", z, p["decoder/dense/kernel"]) + p["decoder/dense/bias"], "g1")
    g2 = relu(mm("dec1.fwd", g1, p["decoder/dense_1/kernel"]) + p["decoder/dense_1/bias"], "g2")
    logits = mm("dec2.fwd", g2, p["decoder/dense_2/kernel"]) + p["decoder/dense_2/bias"]
    elem, dlogit = vo.recon_elem(loss_type, yf, logits)
    recon = elem.sum(axis=1).mean()
    kl_rows = -0.5 * np.sum(1.0 + logvar - mean * mean - np.exp(logvar), axis=1)
    kl_active = np.ones(b, dtype=bool)
    if kl_tolerance > 0:
        floor = kl_tolerance * mean.shape[1]
        kl_active = kl_rows >= floor
        kl_rows = np.maximum(kl_rows, floor)
    kl = kl_rows.mean()
    out = dict(mean=mean, logvar=logvar, z=z, logits=logits, recon=recon, kl=kl, loss=recon + beta * kl)
    g = {}
    gl = dlogit / b
    g["decoder/dense_2/kernel"] = mm("dec2.wgrad", g2.T, gl); g["decoder/dense_2/bias"] = gl.sum(axis=0)
    d = mm("dec2.dgrad", gl, p["decoder/dense_2/kernel"].T) * active(g2, "g2")
    g["decoder/dense_1/kernel"] = mm("dec1.wgrad", g1.T, d); g["decoder/dense_1/bias"] = d.sum(axis=0)
    d = mm("dec1.dgrad", d, p["decoder/dense_1/kernel"].T) * active(g1, "g1")
    g["decoder/dense/kernel"] = mm("dec.wgrad", z.T, d); g["decoder/dense/bias"] = d.sum(axis=0)
    gz = mm("dec.dgrad", d, p["decoder/dense/kernel"].T)
    klmask = kl_active[:, None].astype(dtype)
    gmean = gz + (beta / b) * mean * klmask
    glogvar = gz * (0.5 * eps * std) + (beta / b) * 0.5 * (np.exp(logvar) - 1.0) * klmask
    g["mean/kernel"] = mm("mean.wgrad", h2.T, gmean); g["mean/bias"] = gmean.sum(axis=0)
    g["logstd_sqare/kernel"] = mm("logvar.wgrad", h2.T, glogvar); g["logstd_sqare/bias"] = glogvar.sum(axis=0)
    d = (mm("mean.dgrad", gmean, p["mean/kernel"].T) + mm("logvar.dgrad", glogvar, p["logstd_sqare/kernel"].T)) * active(h2, "h2")
    g["encoder/dense_1/kernel"] = mm("enc1.wgrad", h1.T, d); g["encoder/dense_1/bias"] = d.sum(axis=0)
    d = mm("enc1.dgrad", d, p["encoder/dense_1/kernel"].T) * active(h1, "h1")
    g["encoder/dense/kernel"] = mm("enc.wgrad", xf.T, d); g["encoder/dense/bias"] = d.sum(axis=0)
    out["grads"] = g
    out["relu_inputs"] = dict(h1=h1, h2=h2, g1=g1, g2=g2)
    return out
