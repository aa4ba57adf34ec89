"""Inputs of the categorical PPO tests (tests/test_ppo_categorical_gpu.py): networks with kink-free trunk biases on their
states, an old policy whose logits differ row by row, taken indices placed away from the clip bounds, rollouts, warm Adam
slots and the float64 / float32 references of tests/ppo_categorical_oracle.py."""
import numpy as np

import ppo_categorical_oracle as pco
import ppo_depth_oracle as pdo
from ppo_cases import _gap_bias, near_clip_bound, warm_adam

S = 67
LR = 1e-4
NVECS = {"2": (2,), "64": (64,), "7x3": (7, 3), "2x2x2x2": (2, 2, 2, 2), "31x33": (31, 33)}
ARCHS = {"default": ((500, 300), (500, 300)), "p64_v64": ((64,), (64,)), "odd": ((33, 7, 65), (31,)),
         "deep": ((64,) * 8, (32,) * 8)}


class MultiDiscrete:
    def __init__(self, nvec):
        self.nvec = np.asarray(nvec)


def make_ppo(model_dir, arch, cats, policy=None, old=None, state_dim=S, **kw):
    from carla_ppo_b200.ppo import PPO
    kw.setdefault("learning_rate", LR)
    kw.setdefault("value_scale", 1.0)
    kw.setdefault("entropy_scale", 0.01)
    kw.setdefault("epsilon", 0.2)
    m = PPO((state_dim,), MultiDiscrete(cats), model_dir=str(model_dir), seed=0, policy_hidden_sizes=arch[0],
            value_hidden_sizes=arch[1], **kw)
    m.init_session(init_logging=False)
    if policy is not None:
        m.set_weights(policy, old if old is not None else policy)
    return m


def _shim(p):
    q = dict(p)
    q["action_mean/kernel"] = p["action_logits/kernel"]
    return q


def kink_free(arch, cats, states, seed, state_dim=S):
    """init_params with every trunk bias placed so that no pre-activation on `states` is near a ReLU kink"""
    q = pdo.place_biases(_shim(pco.init_params(state_dim, cats, arch[0], arch[1], seed=seed)), states, _gap_bias)
    del q["action_mean/kernel"]
    return {k: v.astype(np.float32) for k, v in q.items()}


def relu_margin(p, states):
    return pdo.relu_margin(_shim(p), states)


def f64(q):
    return {k: v.astype(np.float64) for k, v in q.items()}


def make_batch(arch, cats, n, seed, state_dim=S, spread=0.3):
    """(p, old, states, actions, returns, advantages): the old policy's logits differ from the new one's by ~spread per
    logit and row.  The rows are drawn from 5n candidates (the trunk biases placed on all of them): none with a ratio
    within 1e-4 of a clip bound (absolute and relative), taken in turn from below, inside and above the clip range."""
    from ppo_cases import CLIP_HI, CLIP_LO
    rs = np.random.RandomState(seed)
    N = 5 * n
    s = rs.randn(N, state_dim).astype(np.float32)
    p = kink_free(arch, cats, s, seed + 1, state_dim)
    old = {k: v.copy() for k, v in p.items()}
    keep = {}
    pco.forward(f64(p), s.astype(np.float64), keep)
    hnorm = float(np.sqrt(np.mean(np.sum(keep["h"][-1] ** 2, axis=1)))) + 1e-6
    W = p["action_logits/kernel"]
    old["action_logits/kernel"] = (W + rs.randn(*W.shape) * (spread / hnorm)).astype(np.float32)
    old["action_logits/bias"] = (p["action_logits/bias"] + (spread / 3) * rs.randn(W.shape[1])).astype(np.float32)
    a = np.stack([rs.randint(c, size=N) for c in cats], axis=1).astype(np.float32)
    _, value = pco.forward(f64(p), s.astype(np.float64))
    ret = (value + 0.5 + np.abs(rs.randn(N))).astype(np.float32)
    adv = rs.randn(N).astype(np.float32)
    near = lambda r: near_clip_bound(r) | (np.minimum(np.abs(r - CLIP_LO), np.abs(r - CLIP_HI)) < 1e-4)
    for _ in range(10):
        ratio = pco.loss_and_grads(p, old, s, a, ret, adv, cats, want_grads=False)["ratio"]
        bad = near(ratio)
        if not bad.any():
            break
        a[bad] = np.stack([rs.randint(c, size=int(bad.sum())) for c in cats], axis=1)
    ratio = pco.loss_and_grads(p, old, s, a, ret, adv, cats, want_grads=False)["ratio"]
    ok = ~near(ratio)
    groups = [list(np.flatnonzero(ok & (ratio < CLIP_LO))), list(np.flatnonzero(ok & (ratio >= CLIP_LO) & (ratio <= CLIP_HI))),
              list(np.flatnonzero(ok & (ratio > CLIP_HI)))]
    rows = []
    while len(rows) < n and any(groups):
        for g in groups:
            if g and len(rows) < n:
                rows.append(g.pop(0))
    rows = np.asarray(rows)
    return p, old, s[rows], a[rows], ret[rows], adv[rows]


def rollout(arch, cats, T, seed):
    rs = np.random.RandomState(seed)
    s = rs.randn(T, S).astype(np.float32)
    p = kink_free(arch, cats, s, seed + 1)
    a = np.stack([rs.randint(c, size=T) for c in cats], axis=1).astype(np.float32)
    r = rs.rand(T)
    v = rs.randn(T).astype(np.float32)
    d = np.zeros(T, bool)
    d[T // 3] = d[(2 * T) // 3] = True
    return p, (s, a, r, v, d)


def learn_setup(arch, cats, T, epochs, seed):
    from oracle import ppo_oracle as po
    p, data = rollout(arch, cats, T, seed)
    s, a, r, v, d = data
    perms = np.stack([np.random.RandomState(seed + 10 + e).permutation(T) for e in range(epochs)])
    ret, adv_n, _ = po.returns_and_normalised_advantages(r, v, 0.3, d, 0.99, 0.95)
    g = pco.loss_and_grads(p, p, s, a, ret, adv_n, cats, 0.2, 1.0, 0.01)["grads"]
    return p, data, perms, warm_adam(p, g, seed + 2)


def learn_refs(p, cats, data, perms, batch, adam, lr=LR, **kw):
    """((params, records, applied) in float64, the same in float32) of pco.learn from the warm Adam state `adam`."""
    s, a, r, v, d = data

    def run(dtype):
        q = {k: x.astype(dtype) for k, x in p.items()}
        st = dict(m={k: adam[0][k].astype(dtype) for k in p}, v={k: adam[1][k].astype(dtype) for k in p},
                  beta1_power=adam[2][0], beta2_power=adam[2][1])
        rec, applied = pco.learn(q, st, s, a, v, r, d, 0.3, cats, 0.99, 0.95, lr, 0.2, 1.0, 0.01, len(perms), batch,
                                 perms, dtype=dtype, **kw)
        return q, rec, applied
    return run(np.float64), run(np.float32)


def persistent_learn(model_dir, arch_name, nvec_name, T, batch, epochs):
    """learn() of ARCHS[arch_name] over NVECS[nvec_name] (in a fresh process: CPB_PPO_PERSISTENT is read once)."""
    arch, cats = ARCHS[arch_name], NVECS[nvec_name]
    p, data, perms, adam = learn_setup(arch, cats, T, epochs, seed=40)
    m = make_ppo(model_dir, arch, cats, p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    s, a, r, v, d = data
    m._workspace(min(batch, T), T).fill_(0xFF)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=epochs, batch_size=batch, perms=perms, return_metrics=True)
    return m.get_weights(), metrics
