"""Float64 restatement of the PPO at any depth, for both policy heads (cpb_ppo_spec_* and cpb_ppo_cat_*).

A network is a dict of tensors: the dense trunk layers (dense, dense_1, ... in TF creation order: the policy trunk, then
the value trunk), the policy head and the value head.  The architecture is read from the names and shapes.  The head is a
small value passed to every function that needs it:

* a Gaussian head is its action bounds ``(low, high)``: mean = low + (tanh(h W + b) + 1) / 2 (high - low) from
  ``action_mean/*``, and a state-independent ``action_logstd``;
* a categorical head is its tuple of category counts ``(n_1, .., n_K)``: logits z = h W + b from ``action_logits/*``, one
  softmax per component.

At two layers per trunk with a Gaussian head every function performs the operations of oracle.ppo_oracle in the same
order, so the results are bit-identical (tests/test_ppo_depth_cpu.py and tests/test_ppo_learn_options_cpu.py pin that).
Every function takes float64 or float32 (``dtype``)."""
from collections import OrderedDict

import numpy as np

from oracle import ppo_oracle as po
from oracle.vae_oracle import adam_apply


# ------------------------------------------------------------------------------------------------------------- heads
def is_categorical(head):
    """True for a tuple of category counts, False for (low, high) bounds."""
    return np.ndim(head[0]) == 0


def head_names(head):
    """(kernel, bias) of the head's dense layer."""
    return ("action_logits/kernel", "action_logits/bias") if is_categorical(head) else ("action_mean/kernel",
                                                                                        "action_mean/bias")


def offsets(cats):
    return np.concatenate([[0], np.cumsum(cats)]).astype(int)


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


def categorical_log_prob(lp, a, cats):
    off = offsets(cats)
    a = np.asarray(a).astype(int)
    rows = np.arange(lp.shape[0])
    return sum(lp[rows, off[k] + a[:, k]] for k in range(len(cats)))


def _head_forward(p, h, head, keep):
    """The policy head on the top policy activations h: the Gaussian mean or the logits."""
    kernel, bias = head_names(head)
    if is_categorical(head):
        return h @ p[kernel] + p[bias]
    low, high = head
    t = np.tanh(h @ p[kernel] + p[bias])
    keep["t"] = t
    return low + ((t + 1.0) / 2.0) * (high - low)


def _policy_terms(p, old, out, out_old, a, head):
    """(log-prob of a under p [B, 1] or [B], under old, the entropy term before entropy_scale, what the gradient needs)"""
    if is_categorical(head):
        lp = log_softmax(out, head)
        H = entropy_per_component(lp, head)
        return (categorical_log_prob(lp, a, head), categorical_log_prob(log_softmax(out_old, head), a, head),
                np.mean(H.sum(axis=1)), (lp, H))
    logstd = p["action_logstd"]
    return po.log_prob(out, logstd, a), po.log_prob(out_old, old["action_logstd"], a), np.sum(po.ENTROPY_CONST + logstd), None


def _head_backward(p, keep, out, a, head, dlogp, terms, entropy_scale, bsz, g):
    """d loss / d (head pre-activation) from dlogp = d loss / d logp [B, 1]; action_logstd's gradient into g."""
    if is_categorical(head):
        cats, (lp, H) = head, terms
        pr = np.exp(lp)
        off = offsets(cats)
        onehot = np.zeros_like(out)
        rows = np.arange(bsz)
        for k in range(len(cats)):
            onehot[rows, off[k] + a[:, k].astype(int)] = 1.0
        Hcol = np.concatenate([np.repeat(H[:, k:k + 1], cats[k], axis=1) for k in range(len(cats))], axis=1)
        return dlogp * (onehot - pr) + (entropy_scale / bsz) * pr * (lp + Hcol)
    low, high = head
    std = np.exp(p["action_logstd"])
    diff = (a - out) / std
    dmu = dlogp * diff / std
    g["action_logstd"] = np.sum(dlogp * (diff * diff - 1.0), axis=0) - entropy_scale
    dt = dmu * 0.5 * (high - low)
    return dt * (1.0 - keep["t"] ** 2)


# ------------------------------------------------------------------------------------------------------------ trunks
def dense_name(k, what="kernel"):
    return "dense%s/%s" % ("_%d" % k if k else "", what)


def param_shapes(state_dim, head, policy_sizes, value_sizes):
    """name -> shape in TF creation order: 2P + 2V + 5 tensors (Gaussian) or 2P + 2V + 4 (categorical)."""
    s = OrderedDict()
    P = len(policy_sizes)
    for k, w in enumerate(policy_sizes):
        s[dense_name(k)] = (policy_sizes[k - 1] if k else state_dim, w)
        s[dense_name(k, "bias")] = (w,)
    kernel, bias = head_names(head)
    n = int(sum(head)) if is_categorical(head) else len(head[0])
    s[kernel] = (policy_sizes[-1], n)
    s[bias] = (n,)
    if not is_categorical(head):
        s["action_logstd"] = (n,)
    for j, w in enumerate(value_sizes):
        s[dense_name(P + j)] = (value_sizes[j - 1] if j else state_dim, w)
        s[dense_name(P + j, "bias")] = (w,)
    s["value/kernel"] = (value_sizes[-1], 1)
    s["value/bias"] = (1,)
    return s


def init_params(state_dim, head, policy_sizes, value_sizes, seed=0, initial_std=0.4, dtype=np.float32):
    """PPO._initial_weights at this architecture: glorot-uniform trunk kernels and value kernel, zero biases, the head
    kernel variance_scaling(0.1) truncated normal with fan-in = the last policy width, logstd = log(initial_std)."""
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(state_dim, head, policy_sizes, value_sizes).items():
        if name == "action_logstd":
            out[name] = np.full(shape, np.log(initial_std), dtype)
        elif name.endswith("bias"):
            out[name] = np.zeros(shape, dtype)
        elif name == head_names(head)[0]:
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


def architecture(p):
    """(policy_sizes, value_sizes) of a parameter dict in TF creation order: the dense layers before the policy head are
    the policy trunk, the ones after it the value trunk (the shapes alone do not tell them apart when a width equals the
    state size, e.g. state 1 with widths (1, 1))."""
    names = list(p)
    head = names.index("action_logits/kernel" if "action_logits/kernel" in p else "action_mean/kernel")
    pol, val = [], []
    k = 0
    while dense_name(k) in p:
        (pol if names.index(dense_name(k)) < head else val).append(np.shape(p[dense_name(k)])[1])
        k += 1
    return tuple(pol), tuple(val)


def trunk_names(p):
    """([(kernel, bias)] of the policy trunk, [(kernel, bias)] of the value trunk)"""
    pol, val = architecture(p)
    P = len(pol)
    return ([(dense_name(k), dense_name(k, "bias")) for k in range(P)],
            [(dense_name(P + j), dense_name(P + j, "bias")) for j in range(len(val))])


def _trunk(p, s, layers, keep):
    h = s
    for w, b in layers:
        h = np.maximum(h @ p[w] + p[b], 0.0)
        keep.append(h)
    return h


def _trunk_backward(p, s, layers, acts, d, g):
    """d = masked gradient w.r.t. the top layer's output; weight / bias gradients top down into g."""
    for l in range(len(layers) - 1, -1, -1):
        w, b = layers[l]
        below = acts[l - 1] if l else s
        g[w] = below.T @ d
        g[b] = d.sum(axis=0)
        if l:
            d = (d @ p[w].T) * (acts[l - 1] > 0)


def forward(p, s, head, keep=None):
    """-> (Gaussian mean [B, A] or logits [B, N], value [B])"""
    pol, val = trunk_names(p)
    kept = {} if keep is None else keep
    hs, gs = [], []
    h = _trunk(p, s, pol, hs)
    out = _head_forward(p, h, head, kept)
    g = _trunk(p, s, val, gs)
    v = (g @ p["value/kernel"] + p["value/bias"])[:, 0]
    kept.update(h=hs, g=gs)
    return out, v


def predict(p, s, head, noise=None):
    """Gaussian: (mean, or clip(mean + noise sigma) with noise, value).  Categorical: (indices [B, K] int64, value): the
    first largest logit per component, or with noise [B, K] the smallest i with u < cumsum_i p (else the last index)."""
    s = np.asarray(s, np.float64)
    if s.ndim != 2:
        s = s[None]
    out, v = forward(p, s, head)
    if not is_categorical(head):
        low, high = head
        return (out if noise is None else np.clip(out + np.asarray(noise) * np.exp(p["action_logstd"]), low, high)), v
    cats, off = head, offsets(head)
    act = np.zeros((s.shape[0], len(cats)), np.int64)
    lp = log_softmax(out, cats)
    for k in range(len(cats)):
        if noise is None:
            act[:, k] = out[:, off[k]:off[k + 1]].argmax(axis=1)
        else:
            c = np.cumsum(np.exp(lp[:, off[k]:off[k + 1]]), axis=1)
            u = np.asarray(noise, np.float64)[:, k:k + 1]
            hit = u < c
            act[:, k] = np.where(hit.any(axis=1), hit.argmax(axis=1), cats[k] - 1)
    return act, v


def logit_gap(p, s, cats):
    """Smallest difference between the top two logits of any component of any row (float64)"""
    z, _ = forward(p, np.asarray(s, np.float64), cats)
    off = offsets(cats)
    gap = np.inf
    for k in range(len(cats)):
        zk = np.sort(z[:, off[k]:off[k + 1]], axis=1)
        gap = min(gap, float((zk[:, -1] - zk[:, -2]).min()))
    return gap


def cdf_bounds(p, s, cats):
    """[B, K] list of each component's cumulative probabilities (float64): the boundaries of the sampled index"""
    z, _ = forward(p, np.asarray(s, np.float64), cats)
    lp = log_softmax(z, cats)
    off = offsets(cats)
    return [np.cumsum(np.exp(lp[:, off[k]:off[k + 1]]), axis=1) for k in range(len(cats))]


def pre_activations(p, states):
    """Every trunk layer's pre-activation on `states` in float64, the policy trunk's first."""
    s = np.asarray(states, np.float64)
    out = []
    for layers in trunk_names(p):
        h = s
        for w, b in layers:
            z = h @ p[w].astype(np.float64) + p[b]
            out.append(z)
            h = np.maximum(z, 0.0)
    return out


def relu_margin(p, states):
    """Smallest |pre-activation| of every trunk layer on `states` (float64)."""
    return min(float(np.abs(z).min()) for z in pre_activations(p, states))


def place_biases(params, states, gap_bias):
    """params with every trunk bias, layer by layer, chosen by gap_bias (ppo_cases.gap_bias) so that no pre-activation
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


# ------------------------------------------------------------------------------------------------ loss and gradients
def loss_and_grads(params, params_old, s, a, ret, adv, head, epsilon=0.2, value_scale=0.5, entropy_scale=0.01,
                   want_grads=True, dtype=np.float64):
    """loss = -L_clip + value_scale L_V - entropy_scale H and its gradients (oracle.ppo_oracle.loss_and_grads at any
    architecture and either head).  The entropy term is the Gaussian's sum(0.5 log(2 pi e) + logstd), or the mean over
    rows of the categorical entropies summed over the components."""
    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    po_ = {k: np.asarray(v, dtype) for k, v in params_old.items()}
    s = np.asarray(s, dtype); ret = np.asarray(ret, dtype); adv = np.asarray(adv, dtype)
    if is_categorical(head):
        a = np.asarray(a)
    else:
        a = np.asarray(a, dtype)
        head = (np.asarray(head[0], dtype), np.asarray(head[1], dtype))
    bsz = s.shape[0]
    clip_lo, clip_hi = float(np.float32(1.0 - epsilon)), float(np.float32(1.0 + epsilon))
    value_scale, entropy_scale = float(np.float32(value_scale)), float(np.float32(entropy_scale))
    keep = {}
    out, v = forward(p, s, head, keep)
    out_old, _ = forward(po_, s, head)
    logp, logp_old, entropy, terms = _policy_terms(p, po_, out, out_old, a, head)
    ratio = np.exp(logp - logp_old)
    advc = adv.reshape(ratio.shape)
    unclipped = ratio * advc
    clipped = np.clip(ratio, clip_lo, clip_hi) * advc
    policy_loss = np.mean(np.minimum(unclipped, clipped))
    value_loss = np.mean((v - ret) ** 2) * value_scale
    entropy_loss = entropy * entropy_scale
    loss = -policy_loss + value_loss - entropy_loss
    res = {"logits" if is_categorical(head) else "mu": out}
    res.update(value=v, logp=logp, ratio=ratio, policy_loss=policy_loss, value_loss=value_loss,
               entropy_loss=entropy_loss, loss=loss, mean_ratio=ratio.mean())
    if not want_grads:
        return res
    pol, val = trunk_names(p)
    kernel, bias = head_names(head)
    g = {}
    first = unclipped <= clipped
    inside = (ratio >= clip_lo) & (ratio <= clip_hi)
    dratio = np.where(first, advc, np.where(inside, advc, 0.0)) * (-1.0 / bsz)
    dlogp = (dratio * ratio).reshape(-1, 1)
    dpre = _head_backward(p, keep, out, a, head, dlogp, terms, entropy_scale, bsz, g)
    h_top = keep["h"][-1]
    g[kernel] = h_top.T @ dpre
    g[bias] = dpre.sum(axis=0)
    _trunk_backward(p, s, pol, keep["h"], (dpre @ p[kernel].T) * (h_top > 0), g)
    dv = (value_scale * 2.0 / bsz) * (v - ret)
    g_top = keep["g"][-1]
    g["value/kernel"] = g_top.T @ dv[:, None]
    g["value/bias"] = np.array([dv.sum()])
    _trunk_backward(p, s, val, keep["g"], (dv[:, None] @ p["value/kernel"].T) * (g_top > 0), g)
    res["grads"] = g
    return res


# ------------------------------------------------------------------------------------------------------------ guards
def approx_kl(ratio):
    """Stable-Baselines3's approximate KL of the old policy from the new one: mean((r - 1) - log r)."""
    ratio = np.asarray(ratio)
    return np.mean((ratio - 1.0) - np.log(ratio))


def clip_grad_norm(grads, max_norm):
    """torch.nn.utils.clip_grad_norm_ over all tensors of ``grads``: n = sqrt(sum g^2); when max_norm > 0 and
    c = max_norm / (n + 1e-6) < 1 every gradient is multiplied by c.  -> (n, clipped grads); ``grads`` is not changed."""
    norm = np.sqrt(sum(np.sum(np.square(g)) for g in grads.values()))
    if max_norm and max_norm > 0:
        c = max_norm / (norm + 1e-6)
        if c < 1.0:
            return norm, {k: g * c for k, g in grads.items()}
    return norm, dict(grads)


# ------------------------------------------------------------------------------------------------------------- learn
def segmented_gae(rewards, values, bootstrap_values, dones, lengths, gamma, lam):
    """oracle compute_gae on each segment, concatenated; returns = A + V; advantages normalised once over all rows
    (train.py:175-177).  -> (returns, normalised advantages, advantages), float64."""
    offs = np.concatenate([[0], np.cumsum(lengths)]).astype(int)
    adv = np.concatenate([po.compute_gae(np.asarray(rewards)[a:b], np.asarray(values)[a:b], bootstrap_values[s],
                                         np.asarray(dones)[a:b], gamma, lam)
                          for s, (a, b) in enumerate(zip(offs[:-1], offs[1:]))])
    returns = adv + np.asarray(values, np.float64)
    return returns, (adv - adv.mean()) / (adv.std() + 1e-8), adv


def learn(params, adam_state, states, actions, values, rewards, dones, last_value, head,
          gamma=0.99, lam=0.95, lr=1e-4, epsilon=0.2, value_scale=1.0, entropy_scale=0.01,
          num_epochs=3, batch_size=32, perms=None, dtype=np.float64, max_grad_norm=0.0, target_kl=0.0,
          segment_lengths=None, bootstrap_values=None):
    """oracle.ppo_oracle.learn at any architecture and either head, with the guards (0 = off): each minibatch's gradient
    is clipped to the global norm max_grad_norm, and from the first minibatch whose approx_kl exceeds 1.5 * target_kl no
    Adam step is applied.  ``segment_lengths`` / ``bootstrap_values``: the rows are several rollouts
    (cpb_ppo_learn_segments_opts).  ``params`` and ``adam_state`` are updated in place.  -> (records [steps][7]: the five
    losses, approx_kl, the pre-clip norm; NaN rows after the stop, Adam steps applied); with both guards off, columns 0-4
    are ppo_oracle.learn's records."""
    if segment_lengths is None:
        returns, adv_n, _ = po.returns_and_normalised_advantages(rewards, values, last_value, dones, gamma, lam)
    else:
        returns, adv_n, _ = segmented_gae(rewards, values, bootstrap_values, dones, segment_lengths, gamma, lam)
    states = np.asarray(states, dtype)
    actions = np.asarray(actions) if is_categorical(head) else np.asarray(actions, dtype)
    returns32 = returns.astype(np.float32).astype(dtype)        # the float32 feed of the reference
    adv32 = adv_n.astype(np.float32).astype(dtype)
    old = {k: v.copy() for k, v in params.items()}              # update_old_policy()
    n = states.shape[0]
    records, applied, stopped = [], 0, False
    for e in range(num_epochs):
        idx = np.asarray(perms[e])
        for i in range(int(np.ceil(n / batch_size))):
            if stopped:
                records.append((np.nan,) * 7)
                continue
            mb = idx[i * batch_size:(i + 1) * batch_size]
            out = loss_and_grads(params, old, states[mb], actions[mb], returns32[mb], adv32[mb], head, epsilon,
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
