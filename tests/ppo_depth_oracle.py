"""Float64 restatement of oracle/ppo_oracle.py for policy and value trunks of any depth and widths (cpb_ppo_spec).  The
architecture is read from the parameter names (dense, dense_1, ... in TF creation order: the policy trunk, then the
value trunk) and shapes, so one dict of tensors is one network.  At two layers per trunk every function here performs the
operations of oracle.ppo_oracle in the same order, so the results are bit-identical (tests/test_ppo_depth_cpu.py)."""
from collections import OrderedDict

import numpy as np

from oracle import ppo_oracle as po
from oracle.vae_oracle import adam_apply


def dense_name(k, what="kernel"):
    return "dense%s/%s" % ("_%d" % k if k else "", what)


def param_shapes(state_dim, num_actions, policy_sizes, value_sizes):
    """name -> shape in TF creation order: 2P + 2V + 5 tensors."""
    s = OrderedDict()
    P = len(policy_sizes)
    for k, w in enumerate(policy_sizes):
        s[dense_name(k)] = (policy_sizes[k - 1] if k else state_dim, w)
        s[dense_name(k, "bias")] = (w,)
    s["action_mean/kernel"] = (policy_sizes[-1], num_actions)
    s["action_mean/bias"] = (num_actions,)
    s["action_logstd"] = (num_actions,)
    for j, w in enumerate(value_sizes):
        s[dense_name(P + j)] = (value_sizes[j - 1] if j else state_dim, w)
        s[dense_name(P + j, "bias")] = (w,)
    s["value/kernel"] = (value_sizes[-1], 1)
    s["value/bias"] = (1,)
    return s


def architecture(p):
    """(policy_sizes, value_sizes) of a parameter dict: the policy trunk is the chain of dense kernels that ends in the
    action head's input width; the value trunk starts at the next kernel that reads the state."""
    kernels = []
    while dense_name(len(kernels)) in p:
        kernels.append(np.shape(p[dense_name(len(kernels))]))
    S = kernels[0][0]
    for P in range(1, len(kernels)):
        pol, val = kernels[:P], kernels[P:]
        if (all(pol[i][0] == pol[i - 1][1] for i in range(1, P)) and val[0][0] == S
                and pol[-1][1] == np.shape(p["action_mean/kernel"])[0]
                and all(val[i][0] == val[i - 1][1] for i in range(1, len(val)))
                and val[-1][1] == np.shape(p["value/kernel"])[0]):
            return tuple(k[1] for k in pol), tuple(k[1] for k in val)
    raise ValueError("no policy / value split of %r" % (kernels,))


def trunk_names(p):
    """([(kernel, bias)] of the policy trunk, [(kernel, bias)] of the value trunk)"""
    pol, val = architecture(p)
    P = len(pol)
    return ([(dense_name(k), dense_name(k, "bias")) for k in range(P)],
            [(dense_name(P + j), dense_name(P + j, "bias")) for j in range(len(val))])


def init_params(state_dim, num_actions, policy_sizes, value_sizes, seed=0, initial_std=0.4, dtype=np.float32):
    """PPO._initial_weights at this architecture: glorot-uniform trunk kernels and value kernel, zero biases, the
    action_mean kernel variance_scaling(0.1) truncated normal with fan-in = the last policy width, logstd = log(std)."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(state_dim, num_actions, policy_sizes, value_sizes).items():
        if name == "action_logstd":
            out[name] = np.full(shape, np.log(initial_std), dtype)
        elif name.endswith("bias"):
            out[name] = np.zeros(shape, dtype)
        elif name == "action_mean/kernel":
            std = np.sqrt(0.1 / shape[0]) / 0.87962566103423978
            t = rng.randn(*shape)
            bad = np.abs(t) > 2
            while bad.any():
                t[bad] = rng.randn(int(bad.sum()))
                bad = np.abs(t) > 2
            out[name] = (t * std).astype(dtype)
        else:
            limit = np.sqrt(6.0 / (shape[0] + shape[1]))
            out[name] = rng.uniform(-limit, limit, size=shape).astype(dtype)
    return out


def _trunk(p, s, layers, keep):
    h = s
    for w, b in layers:
        h = np.maximum(h @ p[w] + p[b], 0.0)
        keep.append(h)
    return h


def forward(p, s, low, high, keep=None):
    pol, val = trunk_names(p)
    hs, gs = [], []
    h = _trunk(p, s, pol, hs)
    t = np.tanh(h @ p["action_mean/kernel"] + p["action_mean/bias"])
    mu = low + ((t + 1.0) / 2.0) * (high - low)
    g = _trunk(p, s, val, gs)
    v = (g @ p["value/kernel"] + p["value/bias"])[:, 0]
    if keep is not None:
        keep.update(h=hs, g=gs, t=t)
    return mu, v


def predict(p, s, low, high, noise=None):
    s = np.asarray(s, np.float64)
    if s.ndim != 2:
        s = s[None]
    mu, v = forward(p, s, low, high)
    act = mu if noise is None else np.clip(mu + np.asarray(noise) * np.exp(p["action_logstd"]), low, high)
    return act, v


def _trunk_backward(p, s, layers, acts, d, g):
    """d = masked gradient w.r.t. the top layer's output; weight / bias gradients top down into g."""
    for l in range(len(layers) - 1, -1, -1):
        w, b = layers[l]
        below = acts[l - 1] if l else s
        g[w] = below.T @ d
        g[b] = d.sum(axis=0)
        if l:
            d = (d @ p[w].T) * (acts[l - 1] > 0)


def loss_and_grads(params, params_old, s, a, ret, adv, low, high, epsilon=0.2, value_scale=0.5,
                   entropy_scale=0.01, want_grads=True, dtype=np.float64):
    """oracle.ppo_oracle.loss_and_grads at any architecture."""
    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    po_ = {k: np.asarray(v, dtype) for k, v in params_old.items()}
    s = np.asarray(s, dtype); a = np.asarray(a, dtype); ret = np.asarray(ret, dtype); adv = np.asarray(adv, dtype)
    low = np.asarray(low, dtype); high = np.asarray(high, dtype)
    bsz = s.shape[0]
    clip_lo, clip_hi = float(np.float32(1.0 - epsilon)), float(np.float32(1.0 + epsilon))
    value_scale, entropy_scale = float(np.float32(value_scale)), float(np.float32(entropy_scale))
    keep = {}
    mu, v = forward(p, s, low, high, keep)
    mu_old, _ = forward(po_, s, low, high)
    logstd = p["action_logstd"]
    std = np.exp(logstd)
    logp = po.log_prob(mu, logstd, a)
    logp_old = po.log_prob(mu_old, po_["action_logstd"], a)
    ratio = np.exp(logp - logp_old)
    advc = adv[:, None]
    unclipped = ratio * advc
    clipped = np.clip(ratio, clip_lo, clip_hi) * advc
    policy_loss = np.mean(np.minimum(unclipped, clipped))
    value_loss = np.mean((v - ret) ** 2) * value_scale
    entropy_loss = np.sum(po.ENTROPY_CONST + logstd) * entropy_scale
    loss = -policy_loss + value_loss - entropy_loss
    out = dict(mu=mu, value=v, logp=logp, ratio=ratio, policy_loss=policy_loss, value_loss=value_loss,
               entropy_loss=entropy_loss, loss=loss, mean_ratio=ratio.mean())
    if not want_grads:
        return out
    pol, val = trunk_names(p)
    g = {}
    first = unclipped <= clipped
    inside = (ratio >= clip_lo) & (ratio <= clip_hi)
    dratio = np.where(first, advc, np.where(inside, advc, 0.0)) * (-1.0 / bsz)
    dlogp = dratio * ratio
    diff = (a - mu) / std
    dmu = dlogp * diff / std
    g["action_logstd"] = np.sum(dlogp * (diff * diff - 1.0), axis=0) - entropy_scale
    dt = dmu * 0.5 * (high - low)
    dpre = dt * (1.0 - keep["t"] ** 2)
    h_top = keep["h"][-1]
    g["action_mean/kernel"] = h_top.T @ dpre
    g["action_mean/bias"] = dpre.sum(axis=0)
    _trunk_backward(p, s, pol, keep["h"], (dpre @ p["action_mean/kernel"].T) * (h_top > 0), g)
    dv = (value_scale * 2.0 / bsz) * (v - ret)
    g_top = keep["g"][-1]
    g["value/kernel"] = g_top.T @ dv[:, None]
    g["value/bias"] = np.array([dv.sum()])
    _trunk_backward(p, s, val, keep["g"], (dv[:, None] @ p["value/kernel"].T) * (g_top > 0), g)
    out["grads"] = g
    return out


def learn(params, adam_state, states, actions, values, rewards, dones, last_value, low, high,
          gamma=0.99, lam=0.95, lr=1e-4, epsilon=0.2, value_scale=1.0, entropy_scale=0.01,
          num_epochs=3, batch_size=32, perms=None, dtype=np.float64, max_grad_norm=0.0, target_kl=0.0,
          segment_lengths=None, bootstrap_values=None):
    """oracle.ppo_oracle.learn at any architecture, with tests/ppo_options_oracle.py's guards (0 = off) and segments.
    -> (records [steps][7], Adam steps applied); with both guards off, columns 0-4 are ppo_oracle.learn's records."""
    from ppo_options_oracle import approx_kl, clip_grad_norm
    if segment_lengths is None:
        returns, adv_n, _ = po.returns_and_normalised_advantages(rewards, values, last_value, dones, gamma, lam)
    else:
        from ppo_cases import segmented_gae
        returns, adv_n, _ = segmented_gae(rewards, values, bootstrap_values, dones, segment_lengths, gamma, lam)
    states = np.asarray(states, dtype); actions = np.asarray(actions, dtype)
    returns32 = returns.astype(np.float32).astype(dtype)
    adv32 = adv_n.astype(np.float32).astype(dtype)
    old = {k: v.copy() for k, v in params.items()}
    n = states.shape[0]
    records, applied, stopped = [], 0, False
    for e in range(num_epochs):
        idx = np.asarray(perms[e])
        for i in range(int(np.ceil(n / batch_size))):
            if stopped:
                records.append((np.nan,) * 7)
                continue
            mb = idx[i * batch_size:(i + 1) * batch_size]
            out = loss_and_grads(params, old, states[mb], actions[mb], returns32[mb], adv32[mb], low, high,
                                 epsilon, value_scale, entropy_scale, True, dtype)
            kl = approx_kl(out["ratio"])
            norm, grads = clip_grad_norm(out["grads"], max_grad_norm)
            records.append((out["policy_loss"], out["value_loss"], out["entropy_loss"], out["loss"], out["mean_ratio"],
                            kl, norm))
            if target_kl and kl > 1.5 * target_kl:
                stopped = True
                continue
            adam_apply(params, grads, adam_state, lr)
            applied += 1
    return np.asarray(records, np.float64).reshape(-1, 7), applied


def place_biases(params, states, gap_bias):
    """params with every trunk bias, layer by layer, chosen by gap_bias (ppo_cases._gap_bias) so that no pre-activation
    on `states` lies near a ReLU kink."""
    p = {k: v.copy() for k, v in params.items()}
    s = np.asarray(states, np.float64)
    for layers in trunk_names(p):
        h = s
        for w, b in layers:
            z = h @ p[w].astype(np.float64)
            p[b] = gap_bias(z)
            h = np.maximum(z + p[b], 0.0)
    return p


def relu_margin(p, states):
    """Smallest |pre-activation| of every trunk layer on `states` (float64)."""
    s = np.asarray(states, np.float64)
    m = np.inf
    for layers in trunk_names(p):
        h = s
        for w, b in layers:
            z = h @ p[w].astype(np.float64) + p[b]
            m = min(m, float(np.abs(z).min()))
            h = np.maximum(z, 0.0)
    return m
