"""Float64 restatement of the categorical PPO head (cpb_ppo_cat_*, include/carla_ppo_b200.h "Categorical policies") on
top of tests/ppo_depth_oracle.py's trunks: logits z = h_P W + b (action_logits/*), one softmax per component, the clipped
surrogate, value and entropy terms of the loss, their gradients, predict (greedy / inverse-CDF sampling) and the learn
loop with tests/ppo_options_oracle.py's guards.  The categories are read from a parameter dict's shapes together with the
``cats`` argument; every function takes float64 or float32 (``dtype``)."""
from collections import OrderedDict

import numpy as np

import ppo_depth_oracle as pdo
from oracle.vae_oracle import adam_apply


def param_shapes(state_dim, cats, policy_sizes, value_sizes):
    """name -> shape in TF creation order: 2P + 2V + 4 tensors."""
    s = OrderedDict()
    for name, shape in pdo.param_shapes(state_dim, len(cats), policy_sizes, value_sizes).items():
        if name == "action_mean/kernel":
            s["action_logits/kernel"] = (policy_sizes[-1], int(sum(cats)))
        elif name == "action_mean/bias":
            s["action_logits/bias"] = (int(sum(cats)),)
        elif name != "action_logstd":
            s[name] = shape
    return s


def init_params(state_dim, cats, policy_sizes, value_sizes, seed=0, dtype=np.float32):
    """PPO._initial_weights of a categorical agent: glorot trunks, zero biases, the action_logits kernel drawn like
    action_mean's (variance_scaling(0.1) truncated normal)."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(state_dim, cats, policy_sizes, value_sizes).items():
        if name.endswith("bias"):
            out[name] = np.zeros(shape, dtype)
        elif name == "action_logits/kernel":
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


def trunk_names(p):
    """ppo_depth_oracle.trunk_names of a categorical parameter dict."""
    q = dict(p)
    q["action_mean/kernel"] = p["action_logits/kernel"]
    return pdo.trunk_names(q)


def offsets(cats):
    return np.concatenate([[0], np.cumsum(cats)]).astype(int)


def forward(p, s, keep=None):
    """-> (logits [B, N], value [B])"""
    pol, val = trunk_names(p)
    hs, gs = [], []
    h = pdo._trunk(p, s, pol, hs)
    z = h @ p["action_logits/kernel"] + p["action_logits/bias"]
    g = pdo._trunk(p, s, val, gs)
    v = (g @ p["value/kernel"] + p["value/bias"])[:, 0]
    if keep is not None:
        keep.update(h=hs, g=gs)
    return z, v


def log_softmax(z, cats):
    """log p of every logit, one softmax per component (max subtracted)"""
    out = np.empty_like(z)
    off = offsets(cats)
    for k in range(len(cats)):
        zk = z[:, off[k]:off[k + 1]]
        m = zk.max(axis=1, keepdims=True)
        out[:, off[k]:off[k + 1]] = zk - m - np.log(np.exp(zk - m).sum(axis=1, keepdims=True))
    return out


def entropy_per_component(lp, cats):
    """H [B, K]"""
    off = offsets(cats)
    p = np.exp(lp)
    return np.stack([-(p[:, off[k]:off[k + 1]] * lp[:, off[k]:off[k + 1]]).sum(axis=1) for k in range(len(cats))], axis=1)


def log_prob(lp, a, cats):
    off = offsets(cats)
    a = np.asarray(a).astype(int)
    rows = np.arange(lp.shape[0])
    return sum(lp[rows, off[k] + a[:, k]] for k in range(len(cats)))


def predict(p, s, cats, noise=None):
    """-> (indices [B, K] int64, value [B]): the first largest logit per component, or with noise [B, K] the smallest i with
    u < cumsum_i p (else the last index with p > 0)."""
    s = np.asarray(s, np.float64)
    z, v = forward(p, s)
    off = offsets(cats)
    out = np.zeros((s.shape[0], len(cats)), np.int64)
    lp = log_softmax(z, cats)
    for k in range(len(cats)):
        zk = z[:, off[k]:off[k + 1]]
        if noise is None:
            out[:, k] = zk.argmax(axis=1)
        else:
            c = np.cumsum(np.exp(lp[:, off[k]:off[k + 1]]), axis=1)
            u = np.asarray(noise, np.float64)[:, k:k + 1]
            hit = u < c
            out[:, k] = np.where(hit.any(axis=1), hit.argmax(axis=1), cats[k] - 1)
    return out, v


def logit_gap(p, s, cats):
    """Smallest difference between the top two logits of any component of any row (float64)"""
    z, _ = forward(p, np.asarray(s, np.float64))
    off = offsets(cats)
    gap = np.inf
    for k in range(len(cats)):
        zk = np.sort(z[:, off[k]:off[k + 1]], axis=1)
        gap = min(gap, float((zk[:, -1] - zk[:, -2]).min()))
    return gap


def cdf_bounds(p, s, cats):
    """[B, K] list of each component's cumulative probabilities (float64): the boundaries of the sampled index"""
    z, _ = forward(p, np.asarray(s, np.float64))
    lp = log_softmax(z, cats)
    off = offsets(cats)
    return [np.cumsum(np.exp(lp[:, off[k]:off[k + 1]]), axis=1) for k in range(len(cats))]


def loss_and_grads(params, params_old, s, a, ret, adv, cats, epsilon=0.2, value_scale=0.5, entropy_scale=0.01,
                   want_grads=True, dtype=np.float64):
    """loss = -L_pi + L_V - entropy_scale * mean_b H_b and its gradients (ppo_depth_oracle.loss_and_grads with the
    categorical head)."""
    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    po_ = {k: np.asarray(v, dtype) for k, v in params_old.items()}
    s = np.asarray(s, dtype); ret = np.asarray(ret, dtype); adv = np.asarray(adv, dtype)
    a = np.asarray(a)
    bsz = s.shape[0]
    clip_lo, clip_hi = float(np.float32(1.0 - epsilon)), float(np.float32(1.0 + epsilon))
    value_scale, entropy_scale = float(np.float32(value_scale)), float(np.float32(entropy_scale))
    keep = {}
    z, v = forward(p, s, keep)
    z_old, _ = forward(po_, s)
    lp = log_softmax(z, cats)
    logp = log_prob(lp, a, cats)
    logp_old = log_prob(log_softmax(z_old, cats), a, cats)
    H = entropy_per_component(lp, cats)
    ratio = np.exp(logp - logp_old)
    unclipped = ratio * adv
    clipped = np.clip(ratio, clip_lo, clip_hi) * adv
    policy_loss = np.mean(np.minimum(unclipped, clipped))
    value_loss = np.mean((v - ret) ** 2) * value_scale
    entropy_loss = np.mean(H.sum(axis=1)) * entropy_scale
    loss = -policy_loss + value_loss - entropy_loss
    out = dict(logits=z, value=v, logp=logp, ratio=ratio, policy_loss=policy_loss, value_loss=value_loss,
               entropy_loss=entropy_loss, loss=loss, mean_ratio=ratio.mean())
    if not want_grads:
        return out
    pol, val = trunk_names(p)
    g = {}
    first = unclipped <= clipped
    inside = (ratio >= clip_lo) & (ratio <= clip_hi)
    dratio = np.where(first, adv, np.where(inside, adv, 0.0)) * (-1.0 / bsz)
    dlogp = (dratio * ratio)[:, None]
    pr = np.exp(lp)
    off = offsets(cats)
    onehot = np.zeros_like(z)
    rows = np.arange(bsz)
    for k in range(len(cats)):
        onehot[rows, off[k] + a[:, k].astype(int)] = 1.0
    Hcol = np.concatenate([np.repeat(H[:, k:k + 1], cats[k], axis=1) for k in range(len(cats))], axis=1)
    dz = dlogp * (onehot - pr) + (entropy_scale / bsz) * pr * (lp + Hcol)
    h_top = keep["h"][-1]
    g["action_logits/kernel"] = h_top.T @ dz
    g["action_logits/bias"] = dz.sum(axis=0)
    pdo._trunk_backward(p, s, pol, keep["h"], (dz @ p["action_logits/kernel"].T) * (h_top > 0), g)
    dv = (value_scale * 2.0 / bsz) * (v - ret)
    g_top = keep["g"][-1]
    g["value/kernel"] = g_top.T @ dv[:, None]
    g["value/bias"] = np.array([dv.sum()])
    pdo._trunk_backward(p, s, val, keep["g"], (dv[:, None] @ p["value/kernel"].T) * (g_top > 0), g)
    out["grads"] = g
    return out


def learn(params, adam_state, states, actions, values, rewards, dones, last_value, cats,
          gamma=0.99, lam=0.95, lr=1e-4, epsilon=0.2, value_scale=1.0, entropy_scale=0.01,
          num_epochs=3, batch_size=32, perms=None, dtype=np.float64, max_grad_norm=0.0, target_kl=0.0,
          segment_lengths=None, bootstrap_values=None):
    """ppo_depth_oracle.learn with the categorical head.  -> (records [steps][7], Adam steps applied)"""
    from oracle import ppo_oracle as po
    from ppo_options_oracle import approx_kl, clip_grad_norm
    if segment_lengths is None:
        returns, adv_n, _ = po.returns_and_normalised_advantages(rewards, values, last_value, dones, gamma, lam)
    else:
        from ppo_cases import segmented_gae
        returns, adv_n, _ = segmented_gae(rewards, values, bootstrap_values, dones, segment_lengths, gamma, lam)
    states = np.asarray(states, dtype); actions = np.asarray(actions)
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
            out = loss_and_grads(params, old, states[mb], actions[mb], returns32[mb], adv32[mb], cats, epsilon,
                                 value_scale, entropy_scale, True, dtype)
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
