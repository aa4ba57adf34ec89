"""The PPO cases and builders that the PPO tests share: the networks the C ABI accepts and their inputs, the reference
agent's configs[2] rollout, and train.train's parameters over the replay environment.

A network is described once as ``(state_dim, head, policy_sizes, value_sizes)``, the head being the action bounds
``(low, high)`` of a Gaussian policy or the category counts of a categorical one (tests/ppo_restatement.py)."""
from collections import OrderedDict

import numpy as np

import ppo_restatement as pr
from harness import make_conv_vae
from helpers import Box, shipped_ppo, shipped_vae_weights

S = 67                  # the reference agent's state size: z_dim 64 + 3 measurements
LR = 1e-4

# name -> (state_dim, num_actions, hidden1, hidden2).  state_dim = z_dim + measurements (train.py: z_dim any multiple of 4
# in [4, 1024], 0-6 measurements); the small GEMM reads the first-layer reduction in 64-wide chunks.
CASES = OrderedDict([
    ("z4", (7, 2, 500, 300)),               # smallest latent + 3 measurements: one partial chunk
    ("z100_orient", (106, 2, 500, 300)),    # z not a multiple of 64, all 6 measurements
    ("z1024", (1027, 2, 500, 300)),         # largest latent: 17 chunks
    ("a1", (67, 1, 500, 300)),              # one action
    ("a3_z32", (35, 3, 500, 300)),          # three actions, asymmetric bounds
    ("a4", (67, 4, 500, 300)),              # the head kernel's kMaxActions
    ("tiny", (1, 4, 1, 1)),                 # K = 1, one-wide trunks
    ("odd", (65, 3, 33, 31)),               # one over and one under a 32-wide tile
    ("wide", (130, 2, 1024, 512)),          # many tiles per GEMM
])

# name -> (policy_hidden_sizes, value_hidden_sizes) of the Gaussian depth tests (state 67, two actions)
ARCHS = {"p64_v64": ((64,), (64,)), "p256x2_v256x3": ((256, 256), (256, 256, 256)), "odd": ((33, 7, 65), (31,)),
         "deep": ((64,) * 8, (32,) * 8), "one": ((1,), (1,)), "wide": ((2048,), (1024, 1024)),
         "default": ((500, 300), (500, 300))}
# the architectures and action spaces of the categorical tests
CAT_ARCHS = {"default": ((500, 300), (500, 300)), "p64_v64": ((64,), (64,)), "odd": ((33, 7, 65), (31,)),
             "deep": ((64,) * 8, (32,) * 8)}
NVECS = {"2": (2,), "64": (64,), "7x3": (7, 3), "2x2x2x2": (2, 2, 2, 2), "31x33": (31, 33)}

# every action gets its own bounds, so that a mixed-up action index changes the result
LOW4 = np.array([-1.0, 0.0, -2.0, 0.5])
HIGH4 = np.array([1.0, 1.0, 0.5, 3.0])
LOW, HIGH = np.array([-1.0, 0.0]), np.array([1.0, 1.0])     # the reference agent's action bounds
CLIP_LO, CLIP_HI = float(np.float32(0.8)), float(np.float32(1.2))   # the graph's float32 clip constants (epsilon 0.2)
KINK_MARGIN = 1e-4
# make_batch shifts of the old policy that put about a fifth of the rows in each branch of the clipped surrogate
CLIPPED = dict(mean_shift=0.2, logstd_shift=0.05)


def bounds(num_actions):
    return LOW4[:num_actions].copy(), HIGH4[:num_actions].copy()


def shape_net(S_, A, H1, H2):
    """The network of a CASES shape: two layers of H1, H2 in both trunks."""
    return S_, bounds(A), (H1, H2), (H1, H2)


def gauss_net(arch):
    """A Gaussian network of ARCHS: state 67, two actions."""
    return (S, bounds(2)) + tuple(arch)


def cat_net(arch, cats, state_dim=S):
    return (state_dim, tuple(cats)) + tuple(arch)


REFERENCE = (S, (LOW, HIGH), (500, 300), (500, 300))


def gap_bias(z):
    """Per column of z [n, H]: a float32 bias b in the middle of the widest gap of the sorted -z, so that z + b is as far
    from zero as the rows allow.  The gap is looked for where a quarter to three quarters of the rows are active; where
    that window has no usable gap (e.g. a column whose inactive-input rows are all exactly 0), over all interior gaps."""
    n = z.shape[0]
    u = np.sort(-z, axis=0)
    if n < 4:
        return (u[-1] + 0.5).astype(np.float32)       # every row active, 0.5 from the kink
    cols = np.arange(z.shape[1])
    gaps = u[1:] - u[:-1]
    lo, hi = (n - 1) // 4, n - 1 - (n - 1) // 4
    i = lo + np.argmax(gaps[lo:hi], axis=0)
    narrow = gaps[i, cols] < 4 * KINK_MARGIN
    i = np.where(narrow, np.argmax(gaps, axis=0), i)
    return ((u[i, cols] + u[i + 1, cols]) / 2).astype(np.float32)


def kink_free(net, states, seed):
    """init_params with every trunk bias placed so that no pre-activation on `states` is near a ReLU kink"""
    return pr.place_biases(pr.init_params(*net, seed=seed), states, gap_bias)


def f64(q):
    return {k: v.astype(np.float64) for k, v in q.items()}


def clip_groups(ratio, adv):
    """Row masks of the five branches of min(r * adv, clip(r, 0.8, 1.2) * adv)."""
    r, a = np.asarray(ratio).ravel(), np.asarray(adv).ravel()
    below, above = r < CLIP_LO, r > CLIP_HI
    return OrderedDict([("below_pos", below & (a > 0)), ("below_neg", below & (a < 0)),
                        ("above_pos", above & (a > 0)), ("above_neg", above & (a < 0)), ("inside", ~below & ~above)])


def near_clip_bound(ratio):
    """Rows whose ratio lies within 1e-4 relative of a float32 clip bound, where a float32 rounding could flip the branch."""
    r = np.asarray(ratio).ravel()
    return (np.abs(r / CLIP_LO - 1) < 1e-4) | (np.abs(r / CLIP_HI - 1) < 1e-4)


def make_batch(net, n, seed, init_seed=None, mean_shift=0.02, logstd_shift=0.0, spread=0.3):
    """(p, old, states, actions, returns, advantages) for one loss evaluation; p = the network's initial weights drawn
    with init_seed (default seed + 1) and kink-free trunk biases on these states.  Returns lie above each state's value, so the value-bias
    gradient (2 / B) sum(v - ret) cannot cancel: a cancelled sum turns the float32 rounding of v into an arbitrary
    relative error (standard-normal returns cancelled it 126-fold at z100_orient, B = 9).

    Gaussian: old = p with action_mean/bias shifted by +-mean_shift and action_logstd by logstd_shift; actions drawn
    around the midpoint of the two policies' means (clipped to the bounds), so the log-ratio takes both signs.  The default
    mean_shift keeps the ratios near 1 (at 3-4 actions a few rows in a hundred leave the clip range), CLIPPED fills all
    five branches.  Rows whose ratio lands near a clip bound are redrawn.

    Categorical: the old policy's logits differ from the new one's by ~spread per logit and row.  The rows are drawn from
    5n candidates (the trunk biases placed on all of them): none with a ratio within 1e-4 of a clip bound (absolute and
    relative), taken in turn from below, inside and above the clip range."""
    state_dim, head = net[:2]
    init_seed = seed + 1 if init_seed is None else init_seed
    rs = np.random.RandomState(seed)
    if pr.is_categorical(head):
        return _categorical_batch(net, n, rs, init_seed, spread)
    low, high = head
    A = len(low)
    s = rs.randn(n, state_dim).astype(np.float32)
    p = kink_free(net, s, init_seed)
    old = {k: v.copy() for k, v in p.items()}
    old["action_mean/bias"] = (p["action_mean/bias"] + mean_shift * np.array([1.0, -1.0, 1.0, -1.0])[:A]).astype(np.float32)
    old["action_logstd"] = (p["action_logstd"] + logstd_shift).astype(np.float32)
    mu, value = pr.forward(f64(p), s.astype(np.float64), head)
    mu_old, _ = pr.forward(f64(old), s.astype(np.float64), head)
    mid, sigma = (mu + mu_old) / 2, np.exp(p["action_logstd"].astype(np.float64))
    a = np.clip(mid + sigma * rs.randn(n, A), low, high).astype(np.float32)
    ret = (value + 0.5 + np.abs(rs.randn(n))).astype(np.float32)
    adv = rs.randn(n).astype(np.float32)
    for _ in range(20):
        ratio = pr.loss_and_grads(p, old, s, a, ret, adv, head, want_grads=False)["ratio"]
        bad = near_clip_bound(ratio)
        if not bad.any():
            break
        a[bad] = np.clip(mid[bad] + sigma * rs.randn(int(bad.sum()), A), low, high).astype(np.float32)
    return p, old, s, a, ret, adv


def _categorical_batch(net, n, rs, init_seed, spread):
    state_dim, cats = net[:2]
    N = 5 * n
    s = rs.randn(N, state_dim).astype(np.float32)
    p = kink_free(net, s, init_seed)
    old = {k: v.copy() for k, v in p.items()}
    keep = {}
    pr.forward(f64(p), s.astype(np.float64), cats, keep)
    hnorm = float(np.sqrt(np.mean(np.sum(keep["h"][-1] ** 2, axis=1)))) + 1e-6
    W = p["action_logits/kernel"]
    old["action_logits/kernel"] = (W + rs.randn(*W.shape) * (spread / hnorm)).astype(np.float32)
    old["action_logits/bias"] = (p["action_logits/bias"] + (spread / 3) * rs.randn(W.shape[1])).astype(np.float32)
    a = np.stack([rs.randint(c, size=N) for c in cats], axis=1).astype(np.float32)
    _, value = pr.forward(f64(p), s.astype(np.float64), cats)
    ret = (value + 0.5 + np.abs(rs.randn(N))).astype(np.float32)
    adv = rs.randn(N).astype(np.float32)
    near = lambda r: near_clip_bound(r) | (np.minimum(np.abs(r - CLIP_LO), np.abs(r - CLIP_HI)) < 1e-4)
    for _ in range(10):
        ratio = pr.loss_and_grads(p, old, s, a, ret, adv, cats, want_grads=False)["ratio"]
        bad = near(ratio)
        if not bad.any():
            break
        a[bad] = np.stack([rs.randint(c, size=int(bad.sum())) for c in cats], axis=1)
    ratio = pr.loss_and_grads(p, old, s, a, ret, adv, cats, want_grads=False)["ratio"]
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


def loss_refs(p, old, s, a, ret, adv, low, high, epsilon=0.2):
    """float64 oracle and the float32 autograd restatement (whose distance from float64 sets the gradient gates)."""
    import torch
    from oracle import ppo_oracle as po, torch_ref
    ref = po.loss_and_grads(p, old, s, a, ret, adv, low, high, epsilon, 1.0, 0.01)
    ref32 = torch_ref.ppo_loss_and_grads(p, old, s, a, ret, adv, low, high, epsilon, 1.0, 0.01, dtype=torch.float32)
    return ref, ref32


def ppo_config(S_, A, H1, H2):
    from carla_ppo_b200 import _lib
    cfg = _lib.PpoConfig()
    cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = S_, A, H1, H2
    low, high = bounds(max(1, min(A, 4)))
    for k in range(len(low)):
        cfg.action_low[k], cfg.action_high[k] = low[k], high[k]
    cfg.epsilon, cfg.value_scale, cfg.entropy_scale = 0.2, 1.0, 0.01
    return cfg


def make_ppo(model_dir, net=REFERENCE, policy=None, old=None, **kw):
    """The PPO class at this network, its weights set to `policy` / `old` when given."""
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import MultiDiscrete
    state_dim, head, pol, val = net
    space = MultiDiscrete(head) if pr.is_categorical(head) else Box(*head)
    kw.setdefault("learning_rate", LR)
    kw.setdefault("value_scale", 1.0)
    kw.setdefault("entropy_scale", 0.01)
    kw.setdefault("epsilon", 0.2)
    m = PPO((state_dim,), space, model_dir=str(model_dir), seed=0, policy_hidden_sizes=pol, value_hidden_sizes=val, **kw)
    m.init_session(init_logging=False)
    if policy is not None:
        m.set_weights(policy, old if old is not None else policy)
    return m


def warm_adam(params, grads, seed):
    """Adam slots and beta powers of a resumed run, scaled to these gradients: from zero slots the first update is
    lr * g / (|g| + 1e-8), which moves elements with |g| ~ 1e-8 by an arbitrary fraction of lr in any float32 arithmetic."""
    rs = np.random.RandomState(seed)
    m, v = {}, {}
    for k, g in grads.items():
        scale = np.sqrt(np.mean(np.square(g))) + 1e-12
        m[k] = (0.5 * scale * rs.uniform(-1, 1, g.shape)).astype(np.float32)
        v[k] = (np.square(np.abs(g) + scale) * rs.uniform(0.5, 2.0, g.shape)).astype(np.float32)
    return m, v, (float(np.float32(0.9 ** 50)), float(np.float32(0.999 ** 50)))


def rollout(net, T, seed):
    """A rollout of the policy with kink-free trunk biases on its states, terminals in the middle (not at the end):
    Gaussian actions sampled from the policy, categorical ones uniform.  -> (p, (s, a, r, v, d))"""
    state_dim, head = net[:2]
    rs = np.random.RandomState(seed)
    s = rs.randn(T, state_dim).astype(np.float32)
    p = kink_free(net, s, seed + 1)
    if pr.is_categorical(head):
        a = np.stack([rs.randint(c, size=T) for c in head], axis=1).astype(np.float32)
    else:
        low, high = head
        mu, _ = pr.forward(f64(p), s.astype(np.float64), head)
        a = np.clip(mu + np.exp(p["action_logstd"].astype(np.float64)) * rs.randn(T, len(low)), low, high).astype(np.float32)
    r = rs.rand(T)
    v = rs.randn(T).astype(np.float32)
    d = np.zeros(T, bool)
    d[T // 3] = d[(2 * T) // 3] = True
    return p, (s, a, r, v, d)


def learn_setup(net, T, epochs, seed):
    """rollout(net, T, seed), one permutation per epoch, and warm Adam slots scaled to the rollout's gradient."""
    from oracle import ppo_oracle as po
    p, data = rollout(net, T, seed)
    s, a, r, v, d = data
    perms = np.stack([np.random.RandomState(seed + 10 + e).permutation(T) for e in range(epochs)])
    ret, adv_n, _ = po.returns_and_normalised_advantages(r, v, 0.3, d, 0.99, 0.95)
    g = pr.loss_and_grads(p, p, s, a, ret, adv_n, net[1], 0.2, 1.0, 0.01)["grads"]
    return p, data, perms, warm_adam(p, g, seed + 2)


def restate(head, p, adam, data, perms, batch, dtype, lr=LR, last_value=0.3, **kw):
    """ppo_restatement.learn in `dtype` from params p and Adam state adam = (m, v, (beta1_power, beta2_power)) over
    data = (s, a, r, v, d).  -> (params, Adam state, records [steps][7], steps applied)"""
    s, a, r, v, d = data
    q = {k: x.astype(dtype) for k, x in p.items()}
    st = dict(m={k: adam[0][k].astype(dtype) for k in p}, v={k: adam[1][k].astype(dtype) for k in p},
              beta1_power=adam[2][0], beta2_power=adam[2][1])
    rec, applied = pr.learn(q, st, s, a, v, r, d, last_value, head, 0.99, 0.95, lr, 0.2, 1.0, 0.01, len(perms), batch,
                            perms, dtype=dtype, **kw)
    return q, st, rec, applied


def learn_refs(net, p, data, perms, batch, adam, lr=LR, **kw):
    """((params, records, applied) in float64, the same in float32) of the restatement's learn from the Adam state adam."""
    out = []
    for dtype in (np.float64, np.float32):
        q, _, rec, applied = restate(net[1], p, adam, data, perms, batch, dtype, lr, **kw)
        out.append((q, rec, applied))
    return tuple(out)


# a4, T = 2500 in minibatches of 1200: the persistent kernel's head loop deals rows out by gridDim.x * 8 (1056 on a
# 132-SM H100 SXM), so each full minibatch takes that loop round twice
PERSISTENT = ("a4", 2500, 1200, 2)


# ------------------------------------------------------------------------------------------------ configs[2]
def baseline_config3(T=2048, E=4):
    """SURVEY section 8(d) config 3 / BASELINE configs[2]: T=2048 rollout, 4 epochs x 8 minibatches of 256,
    shipped agent ckpt-705 (policy, policy_old, warm Adam slots and beta powers), permutations from RandomState(0)."""
    rs = np.random.RandomState(0)
    states = rs.randn(T, 67).astype(np.float32)
    actions = np.clip(rs.randn(T, 2), LOW, HIGH).astype(np.float32)
    rewards = rs.rand(T)
    values = rs.randn(T).astype(np.float32)
    dones = np.zeros(T, bool); dones[-1] = True
    prs = np.random.RandomState(0)
    perms = np.stack([prs.permutation(T) for _ in range(E)])
    return states, actions, rewards, values, dones, perms


# the bounded-update tests at configs[2]: T = 2048, 4 epochs x 256, from ckpt-705 with its Adam state
T3, E3, B3 = 2048, 4, 256
LR_KL = 1e-3          # large enough that the approximate KL grows from minibatch to minibatch (to ~1e-2)
MARGIN = 1.05         # both sides of a KL crossing stay this far from the stop threshold


def shipped_adam():
    pol, z = shipped_ppo("policy")
    return ({k: z["adam_m/" + k] for k in pol}, {k: z["adam_v/" + k] for k in pol},
            (float(z["beta1_power"]), float(z["beta2_power"])))


def shipped_model(path, lr=LR):
    """The PPO class at ckpt-705: policy, policy_old, warm Adam slots and beta powers."""
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = make_ppo(path, REFERENCE, pol, old, learning_rate=lr)
    m.set_weights(pol, old, *shipped_adam())
    return m


def model_state(m):
    return dict(params=m.params.cpu().numpy(), old=m.params_old.cpu().numpy(), m=m.adam_m.cpu().numpy(),
                v=m.adam_v.cpu().numpy(), powers=m.adam_powers.cpu().numpy())


def segment_rollout(lengths, seed=0):
    """configs[2]-shaped rows over segments: states, actions, rewards, values, dones, bootstrap values, perms."""
    rows = int(np.sum(lengths))
    rs = np.random.RandomState(seed)
    s = rs.randn(rows, 67).astype(np.float32)
    a = np.clip(rs.randn(rows, 2), LOW, HIGH).astype(np.float32)
    r, v, boot, d = segment_inputs(lengths, seed)
    perms = np.stack([np.random.RandomState(seed + 1 + e).permutation(rows) for e in range(E3)])
    return s, a, r, v.astype(np.float32), d, boot, perms


def shipped_restate(data, dtype, max_grad_norm=0.0, target_kl=0.0, lr=LR, lengths=None):
    """The guarded update from ckpt-705 in `dtype`: (params, adam state, records [steps][7], steps applied).  data =
    baseline_config3's (s, a, r, v, d, perms), or segment_rollout's (s, a, r, v, d, boot, perms) with `lengths`."""
    pol, _ = shipped_ppo("policy")
    boot = None if lengths is None else data[5]
    return restate((LOW, HIGH), pol, shipped_adam(), data[:5], data[-1], B3, dtype, lr, max_grad_norm=max_grad_norm,
                   target_kl=target_kl, segment_lengths=lengths, bootstrap_values=boot)


def pick_clip(data, lr=LR, lengths=None):
    """A max_grad_norm at which between a quarter and three quarters of the clipped update's minibatches clip: a multiple
    of the median pre-clip norm of the unclipped update (clipping slows the update, so its norms stay higher)."""
    base = float(np.median(shipped_restate(data, np.float64, lr=lr, lengths=lengths)[2][:, 6]))
    for f in (1.0, 1.5, 2.0, 3.0, 4.0):
        norms = shipped_restate(data, np.float64, max_grad_norm=base * f, lr=lr, lengths=lengths)[2][:, 6]
        if 0.25 <= np.mean(norms > base * f) <= 0.75:
            return base * f
    raise AssertionError("no max_grad_norm clips between 25 and 75 %% of the minibatches (median norm %g)" % base)


def pick_target(kl):
    """(k, target_kl): the first minibatch k >= 2 whose approx_kl exceeds every earlier one by MARGIN^2, and the target
    whose threshold 1.5 * target_kl lies at their geometric mean, so that the update stops at k with MARGIN on both sides."""
    for k in range(2, len(kl)):
        prior = float(np.max(kl[:k]))
        if kl[k] > MARGIN ** 2 * prior and prior > 0:
            return k, float(np.sqrt(kl[k] * prior)) / 1.5
    raise AssertionError("no KL crossing with a %.2f margin in %s" % (MARGIN, kl))


def with_null_options(m):
    """Make m's *_opts calls pass a NULL options pointer (both guards off)."""
    from carla_ppo_b200 import _lib
    call = m._call

    def null_call(name, *args):
        if name.endswith("_opts"):
            args = list(args)
            args[_lib.PROTOTYPES[name][1].index(_lib._PO)] = None
        return call(name, *args)
    m._call = null_call


# ------------------------------------------------------------------------------------------------ N environments
def segment_inputs(lengths, seed=0):
    """rewards, values, dones over the concatenated segments and one bootstrap value per segment.  Every other segment
    ends in a terminal, and a few rows inside segments carry done = 1 (the reference masks their bootstrap term and does
    not reset the accumulation)."""
    rs = np.random.RandomState(seed)
    rows = int(np.sum(lengths))
    rewards, values = rs.rand(rows), rs.randn(rows)
    dones = (rs.rand(rows) < 0.02).astype(np.float64)
    ends = np.cumsum(lengths) - 1
    dones[ends] = np.arange(len(lengths)) % 2 == 0
    return rewards, values, rs.randn(len(lengths)), dones


# ------------------------------------------------------------------------------------------------ train.train
def train_params(name, **over):
    p = dict(learning_rate=1e-4, lr_decay=1.0, discount_factor=0.99, gae_lambda=0.95, ppo_epsilon=0.2, initial_std=0.4,
             value_scale=1.0, entropy_scale=0.01, horizon=16, num_epochs=2, num_episodes=2, batch_size=8,
             vae_model="unused", vae_model_type=None, vae_z_dim=None, synchronous=True, fps=30, action_smoothing=0.0,
             model_name=name, reward_fn="reward_speed_centering_angle_multiply", seed=0, eval_interval=1, record_eval=False,
             logging=False)
    p.update(over)
    return p


def shipped_vae(tmp_path, tag):
    return make_conv_vae(tmp_path, shipped_vae_weights()[0], loss="bce", tag="vae_" + tag, training=False)
