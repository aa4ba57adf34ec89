"""Inputs of the PPO depth tests (tests/test_ppo_depth_gpu.py): networks of any architecture with kink-free trunk biases
on their states, rollouts, warm Adam slots, and the float64 / float32 references of tests/ppo_depth_oracle.py."""
import numpy as np

import ppo_depth_oracle as pdo
from ppo_cases import CLIP_HI, CLIP_LO, KINK_MARGIN, _gap_bias, bounds, near_clip_bound, warm_adam  # noqa: F401

S, A = 67, 2
LR = 1e-4

# name -> (policy_hidden_sizes, value_hidden_sizes)
ARCHS = {"p64_v64": ((64,), (64,)), "p256x2_v256x3": ((256, 256), (256, 256, 256)), "odd": ((33, 7, 65), (31,)),
         "deep": ((64,) * 8, (32,) * 8), "one": ((1,), (1,)), "wide": ((2048,), (1024, 1024)),
         "default": ((500, 300), (500, 300))}


def make_ppo(model_dir, arch, policy=None, old=None, **kw):
    from carla_ppo_b200.ppo import PPO
    from helpers import Box
    low, high = bounds(A)
    kw.setdefault("learning_rate", LR)
    kw.setdefault("value_scale", 1.0)
    kw.setdefault("entropy_scale", 0.01)
    kw.setdefault("epsilon", 0.2)
    m = PPO((S,), Box(low, high), model_dir=str(model_dir), seed=0, policy_hidden_sizes=arch[0],
            value_hidden_sizes=arch[1], **kw)
    m.init_session(init_logging=False)
    if policy is not None:
        m.set_weights(policy, old if old is not None else policy)
    return m


def kink_free(arch, states, seed):
    return pdo.place_biases(pdo.init_params(S, A, arch[0], arch[1], seed=seed), states, _gap_bias)


def make_batch(arch, n, seed, mean_shift=0.02):
    """(p, old, states, actions, returns, advantages) as ppo_cases.make_batch, at any architecture."""
    low, high = bounds(A)
    rs = np.random.RandomState(seed)
    s = rs.randn(n, S).astype(np.float32)
    p = kink_free(arch, s, seed + 1)
    old = {k: v.copy() for k, v in p.items()}
    old["action_mean/bias"] = (p["action_mean/bias"] + mean_shift * np.array([1.0, -1.0])).astype(np.float32)
    f64 = lambda q: {k: v.astype(np.float64) for k, v in q.items()}
    mu, value = pdo.forward(f64(p), s.astype(np.float64), low, high)
    mu_old, _ = pdo.forward(f64(old), s.astype(np.float64), low, high)
    mid, sigma = (mu + mu_old) / 2, np.exp(p["action_logstd"].astype(np.float64))
    a = np.clip(mid + sigma * rs.randn(n, A), low, high).astype(np.float32)
    ret = (value + 0.5 + np.abs(rs.randn(n))).astype(np.float32)
    adv = rs.randn(n).astype(np.float32)
    for _ in range(20):
        ratio = pdo.loss_and_grads(p, old, s, a, ret, adv, low, high, want_grads=False)["ratio"]
        bad = near_clip_bound(ratio)
        if not bad.any():
            break
        a[bad] = np.clip(mid[bad] + sigma * rs.randn(int(bad.sum()), A), low, high).astype(np.float32)
    return p, old, s, a, ret, adv


def rollout(arch, T, seed):
    low, high = bounds(A)
    rs = np.random.RandomState(seed)
    s = rs.randn(T, S).astype(np.float32)
    p = kink_free(arch, s, seed + 1)
    mu, _ = pdo.forward({k: v.astype(np.float64) for k, v in p.items()}, s.astype(np.float64), low, high)
    a = np.clip(mu + np.exp(p["action_logstd"].astype(np.float64)) * rs.randn(T, A), low, high).astype(np.float32)
    r = rs.rand(T)
    v = rs.randn(T).astype(np.float32)
    d = np.zeros(T, bool)
    d[T // 3] = d[(2 * T) // 3] = True
    return p, (s, a, r, v, d)


def learn_setup(arch, T, batch, epochs, seed):
    from oracle import ppo_oracle as po
    p, data = rollout(arch, T, seed)
    s, a, r, v, d = data
    perms = np.stack([np.random.RandomState(seed + 10 + e).permutation(T) for e in range(epochs)])
    ret, adv_n, _ = po.returns_and_normalised_advantages(r, v, 0.3, d, 0.99, 0.95)
    low, high = bounds(A)
    g = pdo.loss_and_grads(p, p, s, a, ret, adv_n, low, high, 0.2, 1.0, 0.01)["grads"]
    return p, data, perms, warm_adam(p, g, seed + 2)


def learn_refs(p, data, perms, batch, adam, lr=LR, **kw):
    """((params, records) in float64, the same in float32) of pdo.learn from the warm Adam state `adam`."""
    s, a, r, v, d = data
    low, high = bounds(A)

    def run(dtype):
        q = {k: x.astype(dtype) for k, x in p.items()}
        st = dict(m={k: adam[0][k].astype(dtype) for k in p}, v={k: adam[1][k].astype(dtype) for k in p},
                  beta1_power=adam[2][0], beta2_power=adam[2][1])
        rec, applied = pdo.learn(q, st, s, a, v, r, d, 0.3, low, high, 0.99, 0.95, lr, 0.2, 1.0, 0.01, len(perms), batch,
                                 perms, dtype=dtype, **kw)
        return q, rec, applied
    return run(np.float64), run(np.float32)


def persistent_learn(model_dir, arch_name, T, batch, epochs):
    """learn() of ARCHS[arch_name] (run in a fresh process: CPB_PPO_PERSISTENT is read once per process)."""
    arch = ARCHS[arch_name]
    p, data, perms, adam = learn_setup(arch, T, batch, epochs, seed=40)
    m = make_ppo(model_dir, arch, p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    s, a, r, v, d = data
    m._workspace(min(batch, T), T).fill_(0xFF)           # every float of the workspace reads as NaN until written
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=epochs, batch_size=batch, perms=perms, return_metrics=True)
    return m.get_weights(), metrics
