"""Bounded PPO updates without a GPU: the float64 restatement of gradient-norm clipping and approximate-KL early stopping,
the C ABI's refusals of bad options and NULL pointers in the three *_opts entry points (no launch), and train.py's flags."""
import ctypes as C
import math

import numpy as np
import pytest

import ppo_restatement as pr
from harness import lib, library_state  # noqa: F401
from ppo_cases import CASES, bounds, learn_setup, ppo_config, shape_net
from ppo_checks import LEGACY_OPTS_ENTRIES, ppo_args


# ------------------------------------------------------------------------------------------------ float64 restatement
@pytest.mark.parametrize("max_norm", [0.05, 0.5, 3.0, 1e6])
def test_clipping_is_torch_clip_grad_norm(max_norm):
    import torch
    rs = np.random.RandomState(1)
    grads = {"a": rs.randn(7, 5), "b": rs.randn(5) * 0.1, "c": rs.randn(3, 2) * 0.01}
    norm, clipped = pr.clip_grad_norm(grads, max_norm)
    ts = [torch.tensor(g, dtype=torch.float64, requires_grad=True) for g in grads.values()]
    for t, g in zip(ts, grads.values()):
        t.grad = torch.tensor(g, dtype=torch.float64)
    ref_norm = torch.nn.utils.clip_grad_norm_(ts, max_norm)
    assert norm == pytest.approx(float(ref_norm), rel=1e-15)
    for t, k in zip(ts, grads):
        assert np.allclose(clipped[k], t.grad.numpy(), rtol=1e-15, atol=0)
    assert all(np.array_equal(clipped[k], grads[k]) for k in grads) == (max_norm >= norm)


def test_clipping_off_and_the_input_untouched():
    g = {"a": np.full(4, 3.0)}
    norm, out = pr.clip_grad_norm(g, 0.0)
    assert norm == 6.0 and np.array_equal(out["a"], g["a"])
    norm, out = pr.clip_grad_norm(g, 1.0)
    assert np.allclose(out["a"], 3.0 / (6.0 + 1e-6)) and np.array_equal(g["a"], np.full(4, 3.0))


def test_approx_kl_estimator():
    e = math.e
    assert pr.approx_kl([1.0, 1.0]) == 0.0
    assert pr.approx_kl([e, 1 / e]) == pytest.approx(((e - 2) + (1 / e)) / 2, rel=1e-15)
    r = np.exp(np.random.RandomState(0).randn(1000) * 0.3)
    kl = pr.approx_kl(r)
    assert kl > 0 and kl == pytest.approx(np.mean(r - 1 - np.log(r)), rel=1e-15)


def _scripted_learn(monkeypatch, kls, target_kl, epochs=2, nmb=3):
    """pr.learn over scripted minibatches: minibatch j has approx_kl kls[j] (ratios {x, x} with (x - 1) - log x = kl)."""
    from scipy.optimize import brentq
    calls, steps = [], []

    def fake_loss(params, old, s, *a, **k):
        j = len(calls)
        calls.append(j)
        x = 1.0 if kls[j] == 0 else brentq(lambda x: (x - 1) - math.log(x) - kls[j], 1.0, 10.0)
        return dict(ratio=np.array([[x], [x]]), policy_loss=float(j), value_loss=0.0, entropy_loss=0.0, loss=0.0,
                    mean_ratio=x, grads={"w": np.array([3.0, 4.0])})

    monkeypatch.setattr(pr, "loss_and_grads", fake_loss)
    monkeypatch.setattr(pr, "adam_apply", lambda p, g, st, lr: steps.append(g["w"].copy()))
    n = nmb * 2
    rec, applied = pr.learn({"w": np.zeros(2)}, {}, np.zeros((n, 1)), np.zeros((n, 1)), np.zeros(n), np.zeros(n),
                            np.zeros(n), 0.0, (np.zeros(1), np.ones(1)), num_epochs=epochs, batch_size=2,
                            perms=[np.arange(n)] * epochs, max_grad_norm=2.5, target_kl=target_kl)
    return rec, applied, calls, steps


def test_kl_stop_rule_on_a_scripted_sequence(monkeypatch):
    # threshold 1.5 * 0.01 = 0.015: minibatch 3 (the first of epoch 2) is the first above it
    kls = [0.001, 0.0145, 0.0149, 0.02, 0.0, 0.0]
    rec, applied, calls, steps = _scripted_learn(monkeypatch, kls, 0.01)
    assert applied == 3 and len(steps) == 3 and calls == [0, 1, 2, 3]
    assert rec.shape == (6, 7)
    assert np.allclose(rec[:4, 5], kls[:4], rtol=1e-9, atol=1e-12)
    assert np.all(rec[:4, 6] == 5.0)                               # the pre-clip norm of (3, 4)
    assert np.isnan(rec[4:]).all() and not np.isnan(rec[:4]).any()  # the stopping row is written, later rows are NaN
    for g in steps:                                               # clipped to 2.5 / (5 + 1e-6) before Adam
        assert np.allclose(g, np.array([3.0, 4.0]) * 2.5 / (5 + 1e-6), rtol=1e-15)


def test_kl_stop_at_the_first_minibatch_and_a_target_that_never_triggers(monkeypatch):
    rec, applied, calls, _ = _scripted_learn(monkeypatch, [0.5] + [0.0] * 5, 0.01)
    assert applied == 0 and calls == [0] and np.isnan(rec[1:]).all() and not np.isnan(rec[0]).any()
    rec, applied, calls, _ = _scripted_learn(monkeypatch, [0.0149] * 6, 0.01)
    assert applied == 6 and calls == list(range(6)) and not np.isnan(rec).any()
    rec, applied, _, _ = _scripted_learn(monkeypatch, [5.0] * 6, 0.0)    # target_kl = 0: no stop
    assert applied == 6


def test_guards_off_are_the_oracle_update_bit_for_bit():
    """pr.learn with both guards 0 is oracle.ppo_oracle.learn: the same parameters, Adam state and loss records."""
    from oracle import ppo_oracle as po
    shape, T, batch, epochs = CASES["odd"], 40, 16, 2
    p, (s, a, r, v, d), perms, (m, vv, powers) = learn_setup(shape_net(*shape), T, epochs, seed=3)
    low, high = bounds(shape[1])

    def run(fn, *head, **kw):
        prm = {k: x.astype(np.float64) for k, x in p.items()}
        st = dict(m={k: m[k].astype(np.float64) for k in p}, v={k: vv[k].astype(np.float64) for k in p},
                  beta1_power=powers[0], beta2_power=powers[1])
        out = fn(prm, st, s, a, v, r, d, 0.3, *head, 0.99, 0.95, 1e-3, 0.2, 1.0, 0.01, epochs, batch, perms, **kw)
        return prm, st, out
    p0, st0, rec0 = run(po.learn, low, high)
    p1, st1, (rec1, applied) = run(pr.learn, (low, high), max_grad_norm=0.0, target_kl=0.0)
    assert applied == epochs * 3
    for k in p0:
        assert np.array_equal(p0[k], p1[k]) and np.array_equal(st0["m"][k], st1["m"][k]), k
        assert np.array_equal(st0["v"][k], st1["v"][k]), k
    assert st0["beta1_power"] == st1["beta1_power"] and st0["beta2_power"] == st1["beta2_power"]
    assert np.array_equal(np.asarray(rec0, np.float64), rec1[:, :5])


# ------------------------------------------------------------------------------------------------ C ABI refusals
BAD_OPTIONS = [(-1.0, 0.0), (0.0, -0.01), (float("nan"), 0.0), (0.0, float("nan")), (float("inf"), 0.0),
               (0.0, float("inf")), (-float("inf"), 0.5)]


def _opts(m, t):
    from carla_ppo_b200 import _lib
    return C.byref(_lib.PpoLearnOptions(m, t))


ENTRIES = [("cpb_ppo_" + e, e, names) for e, names in LEGACY_OPTS_ENTRIES.items()]


@pytest.mark.parametrize("entry, args, _", ENTRIES, ids=[e[0] for e in ENTRIES])
@pytest.mark.parametrize("bad", BAD_OPTIONS, ids=lambda o: "%s_%s" % o)
def test_bad_options_are_refused_without_a_launch(lib, entry, args, _, bad):
    cfg = ppo_config(67, 2, 500, 300)
    before = lib.cpb_launch_count()
    assert getattr(lib, entry)(*ppo_args(args, C.byref(cfg), _opts(*bad))) == -1
    assert lib.cpb_launch_count() == before
    assert b"ppo options" in lib.cpb_last_error()


@pytest.mark.parametrize("entry, args, names", ENTRIES, ids=[e[0] for e in ENTRIES])
def test_null_pointers_are_refused_without_a_launch(lib, entry, args, names):
    cfg = ppo_config(67, 2, 500, 300)
    for name in names:
        for opts in (None, _opts(0.5, 0.01)):
            before = lib.cpb_launch_count()
            assert getattr(lib, entry)(*ppo_args(args, C.byref(cfg), opts, **{name: None})) == -1, name
            assert lib.cpb_launch_count() == before, name


# ------------------------------------------------------------------------------------------------ train.py flags
def test_cli_parses_the_guard_flags(monkeypatch):
    from carla_ppo_b200 import train as train_mod
    seen = []
    monkeypatch.setattr(train_mod, "train", lambda params, *a, **k: seen.append(params))
    train_mod.main(["--model_name", "x"])
    train_mod.main(["--model_name", "x", "--max_grad_norm", "0.5", "--target_kl", "0.01", "--reference_loop"])
    assert seen[0]["max_grad_norm"] is None and seen[0]["target_kl"] is None
    assert seen[1]["max_grad_norm"] == 0.5 and seen[1]["target_kl"] == 0.01 and seen[1]["reference_loop"]


# ------------------------------------------------------------------------------------------------ PPO summaries
class _Writer:
    def __init__(self):
        self.scalars = {}

    def add_scalar(self, name, value, step):
        self.scalars[name] = value


def _summaries(tmp_path, pending, applied):
    import torch
    from carla_ppo_b200.ppo import PPO
    from helpers import Box
    m = PPO((67,), Box([-1.0, 0.0], [1.0, 1.0]), model_dir=str(tmp_path / "ppo"), seed=0)
    m._torch, m._lr_dev, m.train_writer = torch, torch.zeros(1), _Writer()
    m._pending_metrics = [torch.tensor(x, dtype=torch.float32) for x in pending]
    m._pending_applied = [torch.tensor([n], dtype=torch.int32) for n in applied]
    m.write_episodic_summaries()
    assert m.episode_counter == 1 and not m._pending_metrics and not m._pending_applied
    return m.train_writer.scalars


def test_summaries_average_evaluated_rows_only(tmp_path):
    nan = float("nan")
    rows = [[1, 2, 3, 4, 5, 0.01, 10], [3, 4, 5, 6, 7, 0.03, 30], [nan] * 7]
    sc = _summaries(tmp_path, [rows, [5, 6, 7, 8, 9]], [2])      # a stopped learn() and one plain train() step
    assert sc["train_loss/policy"] == pytest.approx(3.0) and sc["train/prob_ratio"] == pytest.approx(7.0)
    assert sc["train/approx_kl"] == pytest.approx(0.02) and sc["train/grad_norm"] == pytest.approx(20.0)
    assert sc["train/updates_applied"] == 3


def test_summaries_without_guards_are_unchanged(tmp_path):
    sc = _summaries(tmp_path, [[[1, 2, 3, 4, 5], [3, 4, 5, 6, 7]]], [])
    assert sc["train_loss/policy"] == pytest.approx(2.0)
    assert not {"train/approx_kl", "train/grad_norm", "train/updates_applied"} & set(sc)
