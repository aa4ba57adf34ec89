"""The PPO at every shape the C ABI accepts, without a GPU: the float64 oracle against torch autograd at each shape of
CASES on inputs where the clipped surrogate takes both branches, the weight initialiser and input builders that
tests/test_ppo_shapes_gpu.py uses, and the parameter layout / workspace queries at A = 1..4 and odd sizes."""
import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import pytest

from helpers import Box, rel_l2

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


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_backward_matches_autograd_with_clipped_rows(case):
    """The hand-written backward of ppo_oracle against an independent torch-autograd derivation at this shape, on a
    minibatch whose rows fill all five branches of the clipped surrogate."""
    from oracle import ppo_oracle as po, torch_ref as tr
    S, A, H1, H2 = CASES[case]
    low, high = bounds(A)
    p, old, s, a, ret, adv = make_batch(init_params(S, A, H1, H2, seed=3), 128, seed=4, **CLIPPED)
    ref = po.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    auto = tr.ppo_loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    groups = clip_groups(ref["ratio"], adv)
    assert all(g.any() for g in groups.values()), {k: int(g.sum()) for k, g in groups.items()}
    for key in ("loss", "policy_loss", "value_loss", "entropy_loss", "mean_ratio"):
        assert abs(ref[key] - auto[key]) < 1e-10, key
    assert set(ref["grads"]) == set(po.PPO_TENSORS)
    for name, g in ref["grads"].items():
        assert g.shape == p[name].shape, name
        assert rel_l2(g, auto["grads"][name]) < 1e-10, name


@pytest.mark.parametrize("case", ["a1", "a4", "tiny", "odd"])
def test_initialiser_follows_the_ppo_class(tmp_path, case):
    """init_params draws what PPO._initial_weights draws for the same seed and shapes (the class reads its shapes from
    cpb_ppo_layout, which only needs the session; they are set directly here)."""
    from carla_ppo_b200.ppo import PPO
    from oracle.ppo_oracle import param_shapes
    S, A, H1, H2 = CASES[case]
    m = PPO((S,), Box(*bounds(A)), model_dir=str(tmp_path / "ppo"), seed=7)
    shapes = param_shapes(S, A, (H1, H2), (H1, H2))
    m._names, m._shapes = list(shapes), dict(shapes)
    got, ref = m._initial_weights(), init_params(S, A, H1, H2, seed=7)
    assert list(got) == list(ref)
    for k in ref:
        assert got[k].dtype == ref[k].dtype and np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("case", list(CASES))
def test_biases_keep_pre_activations_off_the_relu_kink(case):
    S, A, H1, H2 = CASES[case]
    for batch in (1, 9, 256):
        p, _, s = make_batch(init_params(S, A, H1, H2), batch, seed=batch)[:3]
        assert relu_margin(p, s) > KINK_MARGIN, batch
        if batch >= 4:                                          # every unit active on some rows and off on others
            for z in pre_activations(p, s):
                assert (z > 0).any(axis=0).all() and (z < 0).any(axis=0).all(), batch


@pytest.fixture(scope="module")
def lib():
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


def _cfg(S, A, H1, H2):
    from carla_ppo_b200 import _lib
    cfg = _lib.PpoConfig()
    cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = S, A, H1, H2
    low, high = bounds(max(1, min(A, 4)))
    for k in range(len(low)):
        cfg.action_low[k], cfg.action_high[k] = low[k], high[k]
    cfg.epsilon, cfg.value_scale, cfg.entropy_scale = 0.2, 1.0, 0.01
    return cfg


LAYOUT_SHAPES = list(CASES.values()) + [(67, 1, 500, 300), (67, 3, 500, 300), (2, 4, 3, 2), (1030, 1, 1, 7)]


@pytest.mark.parametrize("shape", LAYOUT_SHAPES, ids=["S%d_A%d_%dx%d" % s for s in LAYOUT_SHAPES])
def test_layout_matches_oracle_shapes(lib, shape):
    from oracle.ppo_oracle import param_shapes, PPO_TENSORS
    S, A, H1, H2 = shape
    cfg = _cfg(*shape)
    n = lib.cpb_ppo_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (2 * n))(); total = C.c_int64()
    assert lib.cpb_ppo_layout(C.byref(cfg), offs, sizes, shapes, C.byref(total)) == 0
    ref = param_shapes(S, A, (H1, H2), (H1, H2))
    assert [lib.cpb_ppo_tensor_name(i).decode() for i in range(n)] == PPO_TENSORS == list(ref)
    spans = []
    for i, name in enumerate(PPO_TENSORS):
        assert tuple(v for v in shapes[2 * i:2 * i + 2] if v > 0) == ref[name], name
        assert sizes[i] == int(np.prod(ref[name])), name
        assert offs[i] % 64 == 0, name
        spans.append((offs[i], offs[i] + sizes[i]))
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))      # creation order, no overlap
    assert total.value % 64 == 0 and spans[-1][1] <= total.value < spans[-1][1] + 64


@pytest.mark.parametrize("bad", [dict(A=0), dict(A=5), dict(S=0), dict(H1=0), dict(H2=0), dict(A=-1), dict(S=-3)],
                         ids=lambda d: "_".join("%s%d" % kv for kv in d.items()))
def test_layout_and_workspace_refuse_bad_shapes(lib, bad):
    from carla_ppo_b200 import _lib
    shape = dict(S=67, A=2, H1=500, H2=300)
    shape.update(bad)
    cfg = _cfg(shape["S"], shape["A"], shape["H1"], shape["H2"])
    total = C.c_int64(-7)
    assert lib.cpb_ppo_layout(C.byref(cfg), None, None, None, C.byref(total)) == -1      # CPB_ERR_INVALID_ARGUMENT
    assert total.value == -7                                                             # nothing written
    assert lib.cpb_ppo_workspace_bytes(C.byref(cfg), 64, 0) == -1
    with pytest.raises(_lib.CpbError):
        _lib.check(lib.cpb_ppo_layout(C.byref(cfg), None, None, None, None), "cpb_ppo_layout")


def test_workspace_grows_with_batch_and_horizon(lib):
    for shape in (CASES["a4"], CASES["tiny"], CASES["wide"]):
        cfg = C.byref(_cfg(*shape))
        # sizes are rounded up to an alignment, so neighbouring batch sizes may share one
        by_batch = [lib.cpb_ppo_workspace_bytes(cfg, b, 0) for b in (1, 2, 9, 256, 8192, 8200, 20000)]
        assert by_batch[0] > 0 and all(x <= y for x, y in zip(by_batch, by_batch[1:])), by_batch
        assert by_batch[0] < by_batch[3] < by_batch[4] < by_batch[5] < by_batch[6], by_batch
        base = lib.cpb_ppo_workspace_bytes(cfg, 64, 0)
        # the horizon (learn(): T rows of old-policy activations, returns, advantages) only counts beyond max_batch
        assert lib.cpb_ppo_workspace_bytes(cfg, 64, 64) == lib.cpb_ppo_workspace_bytes(cfg, 64, 10) == base
        by_horizon = [lib.cpb_ppo_workspace_bytes(cfg, 64, t) for t in (65, 300, 2500, 4097)]
        assert base <= by_horizon[0] and all(x <= y for x, y in zip(by_horizon, by_horizon[1:])), by_horizon
        assert base < by_horizon[1] < by_horizon[2] < by_horizon[3], by_horizon
        assert lib.cpb_ppo_workspace_bytes(cfg, 0, 0) == -1
        assert lib.cpb_ppo_workspace_bytes(cfg, 64, -1) == -1
    big = lib.cpb_ppo_workspace_bytes(C.byref(_cfg(*CASES["wide"])), 8200, 8200)
    assert 0 < big < 1 << 30
