"""The PPO cases and builders that the PPO tests share: the shapes the C ABI accepts and their inputs, the reference
agent's configs[2] rollout, the segmented GAE in float64, and train.train's parameters over the replay environment."""
from collections import OrderedDict

import numpy as np

from harness import make_conv_vae
from helpers import Box, shipped_vae_weights

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

# every action gets its own bounds, so that a mixed-up action index changes the result
LOW4 = np.array([-1.0, 0.0, -2.0, 0.5])
HIGH4 = np.array([1.0, 1.0, 0.5, 3.0])
CLIP_LO, CLIP_HI = float(np.float32(0.8)), float(np.float32(1.2))   # the graph's float32 clip constants (epsilon 0.2)
KINK_MARGIN = 1e-4
# make_batch shifts of the old policy that put about a fifth of the rows in each branch of the clipped surrogate
CLIPPED = dict(mean_shift=0.2, logstd_shift=0.05)


def bounds(num_actions):
    return LOW4[:num_actions].copy(), HIGH4[:num_actions].copy()


def init_params(state_dim, num_actions, hidden1, hidden2, seed=0, initial_std=0.4):
    """PPO._initial_weights at any (S, A, H1, H2): glorot-uniform kernels, zero biases, the action-mean kernel from
    variance_scaling(0.1) truncated normal, action_logstd = log(initial_std); same RandomState draws in the same order."""
    from oracle.ppo_oracle import param_shapes
    rng = np.random.RandomState(seed)
    out = OrderedDict()
    for name, shape in param_shapes(state_dim, num_actions, (hidden1, hidden2), (hidden1, hidden2)).items():
        if name == "action_logstd":
            out[name] = np.full(shape, np.log(initial_std), np.float32)
        elif name.endswith("bias"):
            out[name] = np.zeros(shape, np.float32)
        elif name == "action_mean/kernel":
            std = np.sqrt(0.1 / shape[0]) / 0.87962566103423978
            t = rng.randn(*shape)
            bad = np.abs(t) > 2
            while bad.any():
                t[bad] = rng.randn(int(bad.sum()))
                bad = np.abs(t) > 2
            out[name] = (t * std).astype(np.float32)
        else:
            limit = np.sqrt(6.0 / (shape[0] + shape[1]))
            out[name] = rng.uniform(-limit, limit, size=shape).astype(np.float32)
    return out


TRUNKS = (("dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias"),
          ("dense_2/kernel", "dense_2/bias", "dense_3/kernel", "dense_3/bias"))


def _gap_bias(z):
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


def pre_activations(p, states):
    """The four trunk pre-activations in float64 (the oracle's forward takes no ReLU masks of its own)."""
    s = np.asarray(states, np.float64)
    out = []
    for w1, b1, w2, b2 in TRUNKS:
        z1 = s @ p[w1].astype(np.float64) + p[b1]
        z2 = np.maximum(z1, 0.0) @ p[w2].astype(np.float64) + p[b2]
        out += [z1, z2]
    return out


def relu_margin(p, states):
    return min(float(np.abs(z).min()) for z in pre_activations(p, states))


def place_biases(params, states):
    """params with the four trunk biases chosen so that no pre-activation on `states` lies near a ReLU kink."""
    p = {k: v.copy() for k, v in params.items()}
    s = np.asarray(states, np.float64)
    for w1, b1, w2, b2 in TRUNKS:
        z = s @ p[w1].astype(np.float64)
        p[b1] = _gap_bias(z)
        z = np.maximum(z + p[b1], 0.0) @ p[w2].astype(np.float64)
        p[b2] = _gap_bias(z)
    return p


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


def make_batch(params, batch, seed, mean_shift=0.02, logstd_shift=0.0):
    """(p, old, states, actions, returns, advantages) for one loss evaluation.  p = params with kink-free trunk biases on
    these states; old = p with action_mean/bias shifted by +-mean_shift and action_logstd by logstd_shift; actions drawn
    around the midpoint of the two policies' means (clipped to the bounds), so the log-ratio takes both signs.  The default
    mean_shift keeps the ratios near 1 (at 3-4 actions a few rows in a hundred leave the clip range), CLIPPED fills all
    five branches.  Rows whose ratio lands near a clip bound are redrawn.  Returns lie above each state's value, so the
    value-bias gradient (2 / B) sum(v - ret) cannot cancel: a cancelled sum turns the float32 rounding of v into an
    arbitrary relative error (standard-normal returns cancelled it 126-fold at z100_orient, B = 9)."""
    from oracle import ppo_oracle as po
    S, A = params["dense/kernel"].shape[0], params["action_logstd"].shape[0]
    low, high = bounds(A)
    rs = np.random.RandomState(seed)
    n = batch
    s = rs.randn(n, S).astype(np.float32)
    p = place_biases(params, s)
    old = {k: v.copy() for k, v in p.items()}
    old["action_mean/bias"] = (p["action_mean/bias"] + mean_shift * np.array([1.0, -1.0, 1.0, -1.0])[:A]).astype(np.float32)
    old["action_logstd"] = (p["action_logstd"] + logstd_shift).astype(np.float32)
    mu, value = po.forward({k: v.astype(np.float64) for k, v in p.items()}, s, low, high)
    mu_old, _ = po.forward({k: v.astype(np.float64) for k, v in old.items()}, s, low, high)
    mid, sigma = (mu + mu_old) / 2, np.exp(p["action_logstd"].astype(np.float64))
    a = np.clip(mid + sigma * rs.randn(n, A), low, high).astype(np.float32)
    ret = (value + 0.5 + np.abs(rs.randn(n))).astype(np.float32)
    adv = rs.randn(n).astype(np.float32)
    for _ in range(20):
        ratio = po.loss_and_grads(p, old, s, a, ret, adv, low, high, want_grads=False)["ratio"]
        bad = near_clip_bound(ratio)
        if not bad.any():
            break
        a[bad] = np.clip(mid[bad] + sigma * rs.randn(int(bad.sum()), A), low, high).astype(np.float32)
    return p, old, s, a, ret, adv


def loss_refs(p, old, s, a, ret, adv, low, high, epsilon=0.2):
    """float64 oracle and the float32 autograd restatement (whose distance from float64 sets the gradient gates)."""
    import torch
    from oracle import ppo_oracle as po, torch_ref
    ref = po.loss_and_grads(p, old, s, a, ret, adv, low, high, epsilon, 1.0, 0.01)
    ref32 = torch_ref.ppo_loss_and_grads(p, old, s, a, ret, adv, low, high, epsilon, 1.0, 0.01, dtype=torch.float32)
    return ref, ref32


def ppo_config(S, A, H1, H2):
    from carla_ppo_b200 import _lib
    cfg = _lib.PpoConfig()
    cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = S, A, H1, H2
    low, high = bounds(max(1, min(A, 4)))
    for k in range(len(low)):
        cfg.action_low[k], cfg.action_high[k] = low[k], high[k]
    cfg.epsilon, cfg.value_scale, cfg.entropy_scale = 0.2, 1.0, 0.01
    return cfg


LOW, HIGH = np.array([-1.0, 0.0]), np.array([1.0, 1.0])     # the reference agent's action bounds


def make_ppo(tmp_path, policy=None, old=None, shape=None, **kw):
    """The PPO class of the reference agent, or at shape = (S, A, H1, H2) with hidden widths other than its 500 / 300:
    everything but the config is shape-generic (it reads cpb_ppo_layout)."""
    from carla_ppo_b200.ppo import PPO
    cls, state_dim, space = PPO, (67,), Box(LOW, HIGH)
    if shape is not None:
        S, A, H1, H2 = shape

        class ShapedPPO(PPO):
            def _cfg(self):
                cfg = super()._cfg()
                cfg.hidden1, cfg.hidden2 = H1, H2
                return cfg
        cls, state_dim, space = ShapedPPO, (S,), Box(*bounds(A))
    kw.setdefault("learning_rate", 1e-4)
    kw.setdefault("value_scale", 1.0)
    kw.setdefault("entropy_scale", 0.01)
    kw.setdefault("epsilon", 0.2)
    m = cls(state_dim, space, model_dir=str(tmp_path / "ppo"), seed=0, **kw)
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


def policy_rollout(shape, T, seed):
    """A rollout of the policy with kink-free trunk biases on its states, terminals in the middle (not at the end)."""
    S, A = shape[:2]
    low, high = bounds(A)
    rs = np.random.RandomState(seed)
    s = rs.randn(T, S).astype(np.float32)
    p = place_biases(init_params(*shape, seed=seed + 1), s)
    from oracle import ppo_oracle as po
    mu, _ = po.forward({k: v.astype(np.float64) for k, v in p.items()}, s, low, high)
    a = np.clip(mu + np.exp(p["action_logstd"].astype(np.float64)) * rs.randn(T, A), low, high).astype(np.float32)
    r = rs.rand(T)
    v = rs.randn(T).astype(np.float32)
    d = np.zeros(T, bool)
    d[T // 3] = d[(2 * T) // 3] = True
    return p, s, a, r, v, d


def learn_setup(shape, T, batch, epochs, seed):
    from oracle import ppo_oracle as po
    p, s, a, r, v, d = policy_rollout(shape, T, seed)
    perms = np.stack([np.random.RandomState(seed + 10 + e).permutation(T) for e in range(epochs)])
    ret, adv_n, _ = po.returns_and_normalised_advantages(r, v, 0.3, d, 0.99, 0.95)
    low, high = bounds(shape[1])
    g = po.loss_and_grads(p, p, s, a, ret, adv_n, low, high, 0.2, 1.0, 0.01)["grads"]
    return p, (s, a, r, v, d), perms, warm_adam(p, g, seed + 2)


# a4, T = 2500 in minibatches of 1200: the persistent kernel's head loop deals rows out by gridDim.x * 8 (1056 on a
# 132-SM H100 SXM), so each full minibatch takes that loop round twice
PERSISTENT = ("a4", 2500, 1200, 2)


def persistent_learn(model_dir):
    """learn() at PERSISTENT; run in a fresh process because CPB_PPO_PERSISTENT is read once per process."""
    case, T, batch, epochs = PERSISTENT
    p, data, perms, adam = learn_setup(CASES[case], T, batch, epochs, seed=30)
    m = make_ppo(model_dir, p, shape=CASES[case])
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    s, a, r, v, d = data
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=epochs, batch_size=batch, perms=perms, return_metrics=True)
    return m.get_weights(), metrics


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


# ------------------------------------------------------------------------------------------------ N environments
def segmented_gae(rewards, values, bootstrap_values, dones, lengths, gamma, lam):
    """oracle compute_gae on each segment, concatenated; returns = A + V; advantages normalised once over all rows
    (train.py:175-177).  -> (returns, normalised advantages, advantages), float64."""
    from oracle import ppo_oracle as po
    offs = np.concatenate([[0], np.cumsum(lengths)]).astype(int)
    adv = np.concatenate([po.compute_gae(np.asarray(rewards)[a:b], np.asarray(values)[a:b], bootstrap_values[s],
                                         np.asarray(dones)[a:b], gamma, lam)
                          for s, (a, b) in enumerate(zip(offs[:-1], offs[1:]))])
    returns = adv + np.asarray(values, np.float64)
    return returns, (adv - adv.mean()) / (adv.std() + 1e-8), adv


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
