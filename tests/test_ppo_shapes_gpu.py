"""GPU parity of the PPO kernels against the float64 oracle at every shape class the C ABI accepts (test_ppo_shapes_cpu.CASES:
state_dim 1..1027, 1-4 actions, hidden widths 1..1024), on minibatches whose rows take both branches of the clipped
surrogate, and for the entry points the PPO class does not reach: cpb_ppo_loss_grad with a row gather, every output of
cpb_gae, the opt-in persistent learn() kernel.

Gates (those of test_ppo_gpu.py): forward quantities 1e-5; gradients max(2 x err32, 2e-5) per tensor and parameters after
Adam steps max(1e-5, 2 x err32), err32 = the float32 restatement's own distance from float64.  Trunk biases are placed so
that no pre-activation lies within 1e-4 of a ReLU kink on the test inputs (the oracle takes no masks of its own)."""
import ctypes as C

import numpy as np
import pytest

from helpers import rel_l2
from ppo_cases import (CASES, CLIPPED, KINK_MARGIN, PERSISTENT, bounds, clip_groups, kink_free, learn_refs, learn_setup,
                       loss_refs, make_batch, make_ppo, near_clip_bound, shape_net, warm_adam)
from ppo_checks import fresh_process
from ppo_restatement import relu_margin

pytestmark = pytest.mark.gpu

TOL = 1e-5
DEFAULT = (67, 2, 500, 300)
POLICY_TENSORS = ("dense/kernel", "dense/bias", "dense_1/kernel", "dense_1/bias", "action_mean/kernel",
                  "action_mean/bias", "action_logstd")
METRICS = ("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio")


class Worst:
    """Asserts err < gate and keeps the check closest to its gate, printed as one 'GATE' line per test."""

    def __init__(self):
        self.err, self.gate, self.what = 0.0, 1.0, ""

    def check(self, err, gate, what):
        assert err < gate, "%s: %.3e (gate %.3e)" % (what, err, gate)
        if err / gate >= self.err / self.gate:
            self.err, self.gate, self.what = err, gate, what

    def report(self, name):
        print("\nGATE %s: worst %s %.3e of gate %.3e" % (name, self.what, self.err, self.gate))


def check_loss(worst, metrics, grads, ref, ref32, label):
    for got, key in zip(metrics, METRICS):
        gate = max(TOL * max(abs(ref[key]), 1e-3), 2 * abs(ref32[key] - ref[key]))
        worst.check(abs(float(got) - ref[key]), gate, "%s %s" % (label, key))
    for name, g in ref["grads"].items():
        assert grads[name].shape == g.shape, name
        gate = max(2 * rel_l2(ref32["grads"][name], g), 2e-5)
        worst.check(rel_l2(grads[name], g), gate, "%s %s" % (label, name))


# ------------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("case", ["tiny", "odd"])
def test_cfg_override_builds_the_constructor_network(tmp_path, case):
    """A PPO subclass that sizes the network through _cfg() (the two-width interface, PPO.init_session) builds what
    the policy_hidden_sizes / value_hidden_sizes arguments build: the same layout, initial weights and workspace."""
    from carla_ppo_b200.ppo import PPO
    from helpers import Box
    S, A, H1, H2 = CASES[case]

    class ShapedPPO(PPO):
        def _cfg(self):
            cfg = super()._cfg()
            cfg.hidden1, cfg.hidden2 = H1, H2
            return cfg
    hook = ShapedPPO((S,), Box(*bounds(A)), model_dir=str(tmp_path / "hook"), seed=0)
    hook.init_session(init_logging=False)
    ctor = make_ppo(tmp_path / "ctor", shape_net(*CASES[case]))
    assert hook.architecture == ctor.architecture == ((H1, H2), (H1, H2))
    assert hook._names == ctor._names and hook._offsets == ctor._offsets and hook._shapes == ctor._shapes
    assert np.array_equal(hook.params.cpu().numpy(), ctor.params.cpu().numpy())
    assert hook._workspace(64, 128).numel() == ctor._workspace(64, 128).numel()


@pytest.mark.parametrize("case", list(CASES))
def test_predict_matches_oracle(tmp_path, case):
    from oracle import ppo_oracle as po
    shape = CASES[case]
    S, A = shape[:2]
    low, high = bounds(A)
    p = kink_free(shape_net(*shape), np.random.RandomState(2).randn(33, S), 1)
    m = make_ppo(tmp_path, shape_net(*shape), p)
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    worst, hit_low, hit_high = Worst(), False, False
    for b in (1, 9, 33):
        s = np.random.RandomState(b).randn(b, S).astype(np.float32)
        act, val = m.predict(s, greedy=True)
        ract, rval = po.predict(p64, s, low, high)
        assert np.shape(act) == np.shape(ract) == ((A,) if b == 1 else (b, A)) and np.shape(val) == np.shape(rval)
        worst.check(rel_l2(act, ract), TOL, "B=%d greedy action" % b)
        worst.check(rel_l2(val, rval), TOL, "B=%d value" % b)
        noise = (3 * np.random.RandomState(100 + b).randn(b, A)).astype(np.float32)    # wide enough to clip both ways
        act, _ = m.predict(s, noise=noise)
        ract, _ = po.predict(p64, s, low, high, noise=noise.astype(np.float64))
        worst.check(rel_l2(act, ract), TOL, "B=%d sampled action" % b)
        assert (act >= low).all() and (act <= high).all()
        hit_low |= bool((ract == low).any())
        hit_high |= bool((ract == high).any())
    assert hit_low and hit_high
    worst.report(case)


# ------------------------------------------------------------------------------------------------- loss / grads
@pytest.mark.parametrize("case", list(CASES))
def test_loss_and_gradients_match_oracle(tmp_path, case):
    shape = CASES[case]
    low, high = bounds(shape[1])
    p, old, s, a, ret, adv = make_batch(shape_net(*shape), 256, 6, init_seed=5)
    assert relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, shape_net(*shape), p, old)
    worst = Worst()
    for b in (1, 8, 9, 256):                # B = 9: one row in the head kernel's second CTA
        metrics, grads = m.loss_and_grads(s[:b], a[:b], ret[:b], adv[:b])
        ref, ref32 = loss_refs(p, old, s[:b], a[:b], ret[:b], adv[:b], low, high)
        assert not near_clip_bound(ref["ratio"]).any()
        check_loss(worst, metrics, grads, ref, ref32, "B=%d" % b)
    worst.report(case)


def test_loss_and_gradients_beyond_8192_rows(tmp_path):
    """B = 8200: cdiv(B, 8) = 1025 head CTAs, more partial sums than the buffer's fixed 1024 rows."""
    low, high = bounds(2)
    p, old, s, a, ret, adv = make_batch(shape_net(*DEFAULT), 8200, 8, init_seed=7)
    assert relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, shape_net(*DEFAULT), p, old)
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    worst = Worst()
    check_loss(worst, metrics, grads, *loss_refs(p, old, s, a, ret, adv, low, high), "B=8200")
    worst.report("B8200")


@pytest.mark.parametrize("case", ["z100_orient", "a4"])
def test_clipped_surrogate_both_branches(tmp_path, case):
    """Rows in all five branches of min(r * adv, clip(r) * adv): below / above the clip range with either sign of the
    advantage, and inside it.  Where the clipped branch is taken the policy gradient of the row is zero."""
    from oracle import ppo_oracle as po
    shape = CASES[case]
    low, high = bounds(shape[1])
    p, old, s, a, ret, adv = make_batch(shape_net(*shape), 256, 10, init_seed=9, **CLIPPED)
    assert relu_margin(p, s) > KINK_MARGIN
    ref, ref32 = loss_refs(p, old, s, a, ret, adv, low, high)
    groups = clip_groups(ref["ratio"], adv)
    assert all(g.mean() >= 0.1 for g in groups.values()), {k: float(g.mean()) for k, g in groups.items()}
    assert not near_clip_bound(ref["ratio"]).any()
    m = make_ppo(tmp_path, shape_net(*shape), p, old)
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    worst = Worst()
    check_loss(worst, metrics, grads, ref, ref32, "clipped")
    # teeth: without clipping the policy gradients are far outside the gates
    free = po.loss_and_grads(p, old, s, a, ret, adv, low, high, 1e9, 1.0, 0.01)
    for name in POLICY_TENSORS:
        gate = max(2 * rel_l2(ref32["grads"][name], ref["grads"][name]), 2e-5)
        assert rel_l2(free["grads"][name], ref["grads"][name]) > 100 * gate, name
    worst.report(case)


@pytest.mark.parametrize("case", ["a3_z32", "odd"])
def test_loss_grad_with_row_gather(tmp_path, case):
    """cpb_ppo_loss_grad with idx: rows idx[i] of states / actions / returns / advantages, repeated and out of order; the
    old policy's log-prob is evaluated on the gathered rows."""
    import torch
    from carla_ppo_b200 import _lib
    shape = CASES[case]
    low, high = bounds(shape[1])
    T, B = 50, 40
    p, old, s, a, ret, adv = make_batch(shape_net(*shape), T, 14, init_seed=13, **CLIPPED)
    idx = np.random.RandomState(15).randint(0, T, B).astype(np.int32)
    assert len(np.unique(idx)) < B and (np.diff(idx) < 0).any() and idx.max() >= B
    m = make_ppo(tmp_path, shape_net(*shape), p, old)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(m._device)
    sd, ad, rd, vd, ixd = dev(s), dev(a), dev(ret), dev(adv), dev(idx)
    metrics = torch.empty(5, dtype=torch.float32, device=m._device)
    ws = m._workspace(B)
    m._call("cpb_ppo_loss_grad", C.byref(m._c), _lib.ptr(m.params), _lib.ptr(m.params_old), _lib.ptr(sd), _lib.ptr(ad),
            _lib.ptr(rd), _lib.ptr(vd), _lib.ptr(ixd), B, _lib.ptr(m.grads), _lib.ptr(metrics), _lib.ptr(ws), ws.numel(),
            m._stream())
    ref, ref32 = loss_refs(p, old, s[idx], a[idx], ret[idx], adv[idx], low, high)
    assert not near_clip_bound(ref["ratio"]).any()
    worst = Worst()
    check_loss(worst, metrics.cpu().numpy(), m.get_grads(), ref, ref32, "gathered")
    worst.report(case)


# ------------------------------------------------------------------------------------------------- Adam steps
def adam_restate(p, slots, powers, steps, dtype):
    """Copies of params and Adam state in `dtype`; `steps(q, st)` advances them."""
    q = {k: x.astype(dtype) for k, x in p.items()}
    st = dict(m={k: slots[0][k].astype(dtype) for k in p}, v={k: slots[1][k].astype(dtype) for k in p},
              beta1_power=powers[0], beta2_power=powers[1])
    rec = steps(q, st)
    return q, rec


@pytest.mark.parametrize("case", ["a3_z32", "tiny"])
def test_two_train_steps_match_oracle(tmp_path, case):
    from oracle import ppo_oracle as po, vae_oracle as vo
    shape = CASES[case]
    low, high = bounds(shape[1])
    p, old, s, a, ret, adv = make_batch(shape_net(*shape), 64, 18, init_seed=17, **CLIPPED)
    assert relu_margin(p, s) > KINK_MARGIN
    m_, v_, powers = warm_adam(p, po.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)["grads"], 19)
    m = make_ppo(tmp_path, shape_net(*shape), p, old)
    m.set_weights(p, old, m_, v_, powers)
    for _ in range(2):
        m.train(s, a, ret, adv)

    def steps(dtype):
        def run(q, st):
            for _ in range(2):
                out = po.loss_and_grads(q, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01, dtype=dtype)
                vo.adam_apply(q, out["grads"], st, 1e-4)
        return adam_restate(p, (m_, v_), powers, run, dtype)[0]
    p64, p32 = steps(np.float64), steps(np.float32)
    got, worst = m.get_weights(), Worst()
    for name in p64:
        worst.check(rel_l2(got[name], p64[name]), max(TOL, 2 * rel_l2(p32[name], p64[name])), name)
    assert m.get_train_step_idx() == 2
    worst.report(case)


def worst_learn(worst, got, metrics, refs, label):
    (p64, rec64, _), (p32, rec32, _) = refs
    rec64, rec32 = rec64[:, :5], rec32[:, :5]
    for name in p64:
        worst.check(rel_l2(got[name], p64[name]), max(TOL, 2 * rel_l2(p32[name], p64[name])), "%s %s" % (label, name))
    assert metrics.shape == rec64.shape
    for col in range(5):
        gate = max(TOL, 2 * rel_l2(rec32[:, col], rec64[:, col]))
        worst.check(rel_l2(metrics[:, col], rec64[:, col]), gate, "%s metric %s" % (label, METRICS[col]))


LEARN = {"a3_z32": (300, 64, 3),        # short last minibatch (300 = 4 x 64 + 44)
         "z1024": (129, 200, 2),        # minibatch larger than T: one minibatch per epoch
         "tiny": (40, 1, 2)}            # one row per minibatch


@pytest.mark.parametrize("case", list(LEARN))
def test_learn_matches_oracle(tmp_path, case):
    shape = CASES[case]
    T, batch, epochs = LEARN[case]
    p, data, perms, adam = learn_setup(shape_net(*shape), T, epochs, 20)
    assert relu_margin(p, data[0]) > KINK_MARGIN
    m = make_ppo(tmp_path, shape_net(*shape), p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    s, a, r, v, d = data
    metrics = m.learn(s, a, v, r, d, 0.3, gamma=0.99, lam=0.95, num_epochs=epochs, batch_size=batch, perms=perms,
                      return_metrics=True)
    worst = Worst()
    worst_learn(worst, m.get_weights(), metrics, learn_refs(shape_net(*shape), p, data, perms, batch, adam), case)
    gold = m.get_old_weights()
    assert all(np.array_equal(gold[k], p[k]) for k in p)                  # theta_old == theta at learn() entry
    assert m.get_train_step_idx() == epochs * -(-T // batch)
    worst.report(case)


def test_persistent_learn_kernel_matches_oracle(tmp_path):
    case, T, batch, epochs = PERSISTENT
    net = shape_net(*CASES[case])
    outs = fresh_process(tmp_path, [(case, net, ("rollout", T, epochs, batch, 30), {})])
    p, data, perms, adam = learn_setup(net, T, epochs, 30)
    assert relu_margin(p, data[0]) > KINK_MARGIN
    refs = learn_refs(net, p, data, perms, batch, adam)
    w = [{k: o[case + ":w:" + k] for k in p} for o in outs]
    worst = Worst()
    for flag, o, wo in zip("01", outs, w):
        worst_learn(worst, wo, o[case + ":metrics"], refs, "persistent=%s" % flag)
    for k in p:
        assert rel_l2(w[1][k], w[0][k]) < 1e-6, (k, rel_l2(w[1][k], w[0][k]))
    worst.report("persistent")


# -------------------------------------------------------------------------------------------------------- GAE
@pytest.mark.parametrize("T", [1, 1023, 1024, 1025, 4097])
def test_gae_outputs_match_oracle(T):
    """cpb_gae's advantages, returns and normalised advantages (learn() reads only its own float32 copies) around the
    1024-thread scan block; at T = 1 the standard deviation is 0 and the normalised advantage exactly 0."""
    import torch
    from carla_ppo_b200 import _lib
    from oracle import ppo_oracle as po
    lib = _lib.load()
    rs = np.random.RandomState(T)
    r, v = rs.rand(T), rs.randn(T)
    d = (rs.rand(T) < 0.02).astype(np.float64)
    d[T // 2] = d[T // 3] = float(T > 2)
    d[-1] = 0.0
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float64)).cuda()
    rd, vd, dd = dev(r), dev(v), dev(d)
    adv, ret, advn = (torch.full((T,), float("nan"), dtype=torch.float64, device="cuda") for _ in range(3))
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.cpb_gae(_lib.ptr(rd), _lib.ptr(vd), 0.3, _lib.ptr(dd), T, 0.99, 0.95, _lib.ptr(adv), _lib.ptr(ret),
                           _lib.ptr(advn), stream), "cpb_gae")
    adv_only = torch.full((T,), float("nan"), dtype=torch.float64, device="cuda")
    _lib.check(lib.cpb_gae(_lib.ptr(rd), _lib.ptr(vd), 0.3, _lib.ptr(dd), T, 0.99, 0.95, _lib.ptr(adv_only), None, None,
                           stream), "cpb_gae")
    torch.cuda.synchronize()
    ref_ret, ref_advn, ref_adv = po.returns_and_normalised_advantages(r, v, 0.3, d, 0.99, 0.95)
    worst = Worst()
    worst.check(rel_l2(adv.cpu().numpy(), ref_adv), 1e-12, "advantages")
    worst.check(rel_l2(ret.cpu().numpy(), ref_ret), 1e-12, "returns")
    worst.check(rel_l2(advn.cpu().numpy(), ref_advn), 1e-12, "normalised advantages")
    if T == 1:
        assert advn.item() == 0.0 and ref_advn[0] == 0.0
    assert torch.equal(adv_only, adv)
    worst.report("T%d" % T)
