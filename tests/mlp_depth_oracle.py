"""The MlpVAE oracle at any depth (test infrastructure for MlpVAEs that do not have two hidden layers per side).

oracle.vae_oracle's MlpVAE functions are written for the reference's default, two hidden layers per side.  This module
restates them for size lists of any length: build_mlp (reference vae/models.py:283-296) loops over the sizes, so the
variables are encoder/dense, encoder/dense_1, ..., mean, logstd_sqare, decoder/dense, ..., and the output layer
decoder/dense_M.  With two layers per side every function here is the vae_oracle one bit for bit
(tests/test_mlp_depth_cpu.py pins that), so the restatement cannot drift from the oracle unnoticed.  The loss, sampling,
KL and Adam pieces are vae_oracle's own.

loss_and_grads takes two optional arguments the oracle lacks:
  * tc_round (array -> array): applied to both operands of exactly the five frame-wide products -- the first encoder
    layer's forward and weight gradient, the output layer's forward, data gradient and weight gradient.  With
    tf32_oracle.round_tf32 it restates math mode 2 at any depth; at two per side it equals tests/mlp_tf32_oracle.py.
  * relu_masks ({"h0", ..., "h{L-1}", "g0", ..., "g{M-1}"} -> bool arrays): the ReLU activity pattern of each hidden
    layer to use, forward (pre * mask) and backward, instead of the sign of this run's own pre-activations, so that a
    device run and the restatement differentiate the same piecewise-linear function.
torch_loss_and_grads is the independent torch-autograd derivation of the same graph."""
from collections import OrderedDict

import numpy as np

from oracle import vae_oracle as vo


def layer_name(scope, i):
    """tf.layers.dense's default names inside one scope: dense, dense_1, dense_2, ..."""
    return "%s/dense%s" % (scope, "_%d" % i if i else "")


def param_shapes(source_shape=(80, 160, 3), target_channels=3, z_dim=64, encoder_sizes=(512, 256), decoder_sizes=(256, 512)):
    """tf.layers.dense variables in creation order."""
    n_in = int(np.prod(source_shape))
    n_out = source_shape[0] * source_shape[1] * target_channels
    s = OrderedDict()

    def dense(name, n, m):
        s[name + "/kernel"] = (n, m)
        s[name + "/bias"] = (m,)
    widths = [n_in] + list(encoder_sizes)
    for i in range(len(encoder_sizes)):
        dense(layer_name("encoder", i), widths[i], widths[i + 1])
    dense("mean", encoder_sizes[-1], z_dim)
    dense("logstd_sqare", encoder_sizes[-1], z_dim)
    widths = [z_dim] + list(decoder_sizes) + [n_out]
    for j in range(len(decoder_sizes) + 1):
        dense(layer_name("decoder", j), widths[j], widths[j + 1])
    return s


def glorot_init(seed=0, dtype=np.float32, **kw):
    """vo.mlp_glorot_init over param_shapes (same draws in the same order)."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(**kw).items():
        if name.endswith("bias"):
            out[name] = np.zeros(shape, dtype)
        else:
            limit = np.sqrt(6.0 / (shape[0] + shape[1]))
            out[name] = rng.uniform(-limit, limit, size=shape).astype(dtype)
    return out


def _layers(p):
    """Names of the encoder layers and of the decoder layers (the last one: the output layer), from the parameters."""
    n_enc = sum(1 for k in p if k.startswith("encoder/") and k.endswith("/kernel"))
    n_dec = sum(1 for k in p if k.startswith("decoder/") and k.endswith("/kernel"))
    return [layer_name("encoder", i) for i in range(n_enc)], [layer_name("decoder", j) for j in range(n_dec)]


def loss_and_grads(params, x, y, eps, loss_type="mse", beta=1.0, kl_tolerance=0.0, want_grads=True, dtype=np.float64,
                   tc_round=None, relu_masks=None):
    """vo.mlp_loss_and_grads at the depth the parameter names describe; x [B,H,W,3], y [B,H,W,C_t], eps [B,z]."""
    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    x = np.asarray(x, dtype); y = np.asarray(y, dtype); eps = np.asarray(eps, dtype)
    vo.verify_range(x); vo.verify_range(y)
    enc, dec = _layers(p)
    n_enc, n_dec = len(enc), len(dec) - 1

    def mm(a, b, frame_wide=False):
        return tc_round(a) @ tc_round(b) if frame_wide and tc_round is not None else a @ b

    def relu(pre, key):
        return np.maximum(pre, 0.0) if relu_masks is None else pre * relu_masks[key]

    def active(act, key):
        return (act > 0) if relu_masks is None else relu_masks[key]

    b = x.shape[0]
    xf = x.reshape(b, -1); yf = y.reshape(b, -1)
    h = []
    for i, name in enumerate(enc):
        h.append(relu(mm(h[-1] if i else xf, p[name + "/kernel"], i == 0) + p[name + "/bias"], "h%d" % i))
    mean = h[-1] @ p["mean/kernel"] + p["mean/bias"]
    logvar = h[-1] @ p["logstd_sqare/kernel"] + p["logstd_sqare/bias"]
    std = np.exp(0.5 * logvar)
    z = mean + eps * std
    g = []
    for j, name in enumerate(dec[:-1]):
        g.append(relu((g[-1] if j else z) @ p[name + "/kernel"] + p[name + "/bias"], "g%d" % j))
    logits = mm(g[-1], p[dec[-1] + "/kernel"], True) + p[dec[-1] + "/bias"]
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
    if not want_grads:
        return out
    gr = {}
    gl = dlogit / b
    gr[dec[-1] + "/kernel"] = mm(g[-1].T, gl, True); gr[dec[-1] + "/bias"] = gl.sum(axis=0)
    d = mm(gl, p[dec[-1] + "/kernel"].T, True) * active(g[-1], "g%d" % (n_dec - 1))
    for j in range(n_dec - 1, 0, -1):
        gr[dec[j] + "/kernel"] = g[j - 1].T @ d; gr[dec[j] + "/bias"] = d.sum(axis=0)
        d = (d @ p[dec[j] + "/kernel"].T) * active(g[j - 1], "g%d" % (j - 1))
    gr[dec[0] + "/kernel"] = z.T @ d; gr[dec[0] + "/bias"] = d.sum(axis=0)
    gz = d @ p[dec[0] + "/kernel"].T
    klmask = kl_active[:, None].astype(dtype)
    gmean = gz + (beta / b) * mean * klmask
    glogvar = gz * (0.5 * eps * std) + (beta / b) * 0.5 * (np.exp(logvar) - 1.0) * klmask
    gr["mean/kernel"] = h[-1].T @ gmean; gr["mean/bias"] = gmean.sum(axis=0)
    gr["logstd_sqare/kernel"] = h[-1].T @ glogvar; gr["logstd_sqare/bias"] = glogvar.sum(axis=0)
    d = (gmean @ p["mean/kernel"].T + glogvar @ p["logstd_sqare/kernel"].T) * active(h[-1], "h%d" % (n_enc - 1))
    for i in range(n_enc - 1, 0, -1):
        gr[enc[i] + "/kernel"] = h[i - 1].T @ d; gr[enc[i] + "/bias"] = d.sum(axis=0)
        d = (d @ p[enc[i] + "/kernel"].T) * active(h[i - 1], "h%d" % (i - 1))
    gr[enc[0] + "/kernel"] = mm(xf.T, d, True); gr[enc[0] + "/bias"] = d.sum(axis=0)
    out["grads"] = gr
    return out


def train_step(params, state, x, y, eps, lr=1e-4, loss_type="mse", beta=1.0, kl_tolerance=0.0, dtype=np.float64, **kw):
    """vo.mlp_train_step at any depth: params / state updated in place; returns (recon, kl)."""
    out = loss_and_grads(params, x, y, eps, loss_type, beta, kl_tolerance, True, dtype, **kw)
    vo.adam_apply(params, out["grads"], state, lr)
    return out["recon"], out["kl"]


def torch_loss_and_grads(params, x, y, eps, loss_type="mse", beta=1.0, kl_tolerance=0.0):
    """The same graph with stock torch ops + autograd in float64: the independent check of the hand-derived backward."""
    import torch
    import torch.nn.functional as F
    p = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in params.items()}
    xt, yt, et = (torch.as_tensor(np.asarray(a, np.float64)) for a in (x, y, eps))
    enc, dec = _layers(p)
    b = xt.shape[0]
    h = xt.reshape(b, -1)
    for name in enc:
        h = F.relu(h @ p[name + "/kernel"] + p[name + "/bias"])
    mean = h @ p["mean/kernel"] + p["mean/bias"]
    logvar = h @ p["logstd_sqare/kernel"] + p["logstd_sqare/bias"]
    g = mean + et * torch.exp(0.5 * logvar)
    for name in dec[:-1]:
        g = F.relu(g @ p[name + "/kernel"] + p[name + "/bias"])
    lf = g @ p[dec[-1] + "/kernel"] + p[dec[-1] + "/bias"]
    yf = yt.reshape(b, -1)
    if loss_type == "mse":
        elem = (yf - torch.sigmoid(lf)) ** 2
    elif loss_type == "bce":
        elem = F.binary_cross_entropy_with_logits(lf, yf, reduction="none")
    else:
        sg = torch.sigmoid(lf)
        elem = -(yf * torch.log(1e-10 + sg) + (1 - yf) * torch.log(1e-10 + 1 - sg))
    recon = elem.sum(dim=1).mean()
    kl_rows = -0.5 * torch.sum(1.0 + logvar - mean * mean - torch.exp(logvar), dim=1)
    if kl_tolerance > 0:
        kl_rows = torch.maximum(kl_rows, torch.full_like(kl_rows, kl_tolerance * mean.shape[1]))
    kl = kl_rows.mean()
    (recon + beta * kl).backward()
    return dict(mean=mean.detach().numpy(), logvar=logvar.detach().numpy(), logits=lf.detach().numpy(),
                recon=float(recon.detach()), kl=float(kl.detach()), grads={k: v.grad.numpy() for k, v in p.items()})
