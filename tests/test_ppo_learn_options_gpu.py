"""Bounded PPO updates on the H100: cpb_ppo_learn_opts, cpb_ppo_learn_segments_opts and cpb_ppo_train_step_opts (global
gradient-norm clipping, approximate-KL early stopping) against the float64 restatement at BASELINE configs[2], bit-identity
with the original entry points when the guards are off, the persistent kernel, the reference loop and train.train."""
import numpy as np
import pytest

import ppo_cases as oc
from helpers import committed_frames, rel_l2
from ppo_cases import REFERENCE, baseline_config3, shipped_vae, train_params
from ppo_checks import fresh_process

pytestmark = pytest.mark.gpu

TOL = 1e-5
KEYS = ("params", "old", "m", "v", "powers")


def _learn(m, data, lengths=None, **kw):
    if lengths is None:
        s, a, r, v, d, perms = data
        last = 0.3
    else:
        s, a, r, v, d, last, perms = data
    return m.learn(s, a, v, r, d, last, num_epochs=oc.E3, batch_size=oc.B3, perms=perms, return_metrics=True,
                   segment_lengths=lengths, **kw)


def _same_state(x, y):
    for k in KEYS:
        assert np.array_equal(x[k], y[k]), k


def _check_against_oracle(m, rec_dev, data, lengths=None, **guards):
    """params, Adam m and v per tensor and metric columns 0-6 (evaluated rows) vs the float64 restatement, at
    max(1e-5, 2 x the float32 restatement's distance); the same NaN rows and steps applied."""
    p64, st64, rec64, n64 = oc.shipped_restate(data, np.float64, lengths=lengths, **guards)
    p32, st32, rec32, n32 = oc.shipped_restate(data, np.float32, lengths=lengths, **guards)
    assert n32 == n64 and int(m.last_steps_applied.item()) == n64
    got = dict(params=m.get_weights(), m=m._unflatten(m.adam_m), v=m._unflatten(m.adam_v))
    for what, ref, ref32 in (("params", p64, p32), ("m", st64["m"], st32["m"]), ("v", st64["v"], st32["v"])):
        for k in ref:
            gate = max(TOL, 2 * rel_l2(ref32[k], ref[k]))
            err = rel_l2(got[what][k], ref[k])
            assert err < gate, "%s %s: %.3e (gate %.3e)" % (what, k, err, gate)
    assert np.array_equal(np.isnan(rec_dev), np.isnan(rec64))
    ok = ~np.isnan(rec64[:, 0])
    # approx_kl = mean((r - 1) - log r) cancels to ~kl from fp32 terms of size |log r| <= |logp| + |logp_old| < 8: a
    # relative gate would measure that rounding at tiny KL, so the column is held to 8 fp32 ulps of 8 per row
    assert np.max(np.abs(rec_dev[ok, 5] - rec64[ok, 5])) <= 2.0 ** -20, np.max(np.abs(rec_dev[ok, 5] - rec64[ok, 5]))
    for col in (0, 1, 2, 3, 4, 6):
        gate = max(TOL, 2 * rel_l2(rec32[ok, col], rec64[ok, col]))
        assert rel_l2(rec_dev[ok, col], rec64[ok, col]) < gate, (col, rel_l2(rec_dev[ok, col], rec64[ok, col]), gate)
    return rec64, n64


def _powers_after(steps):
    _, _, powers = oc.shipped_adam()
    p = np.array(powers, np.float32)
    for _ in range(steps):
        p = p * np.array([0.9, 0.999], np.float32)
    return p


# ------------------------------------------------------------------------------------------------ 1. guards off
SEGMENTS = [700, 700, 648]


@pytest.mark.parametrize("lengths", [None, SEGMENTS], ids=["learn", "segments"])
def test_guards_off_are_the_original_entry_point_bit_for_bit(tmp_path, lengths):
    data = baseline_config3(oc.T3, oc.E3) if lengths is None else oc.segment_rollout(lengths)
    out = {}
    for tag, kw in (("plain", {}), ("zero", dict(max_grad_norm=0.0, target_kl=0.0)),
                    ("null", dict(max_grad_norm=0.0, target_kl=0.0))):
        m = oc.shipped_model(tmp_path / tag, lr=oc.LR_KL)
        if tag == "null":
            oc.with_null_options(m)
        met = _learn(m, data, lengths, **kw)
        out[tag] = (oc.model_state(m), met, m.last_steps_applied)
    plain = out["plain"]
    assert plain[1].shape == (oc.E3 * 8, 5)
    for tag in ("zero", "null"):
        st, met, applied = out[tag]
        _same_state(st, plain[0])
        assert met.shape == (oc.E3 * 8, 7) and np.array_equal(met[:, :5], plain[1])
        assert int(applied.item()) == oc.E3 * 8 and not np.isnan(met).any()


def test_guards_off_train_step_is_cpb_ppo_train_step_bit_for_bit(tmp_path):
    s, a, r, v, d, perms = baseline_config3(oc.T3, 1)
    rs = np.random.RandomState(3)
    ret, adv = rs.randn(oc.T3).astype(np.float32), rs.randn(oc.T3).astype(np.float32)
    out = {}
    for tag in ("plain", "zero", "null", "stop"):
        m = oc.shipped_model(tmp_path / tag, lr=oc.LR_KL)
        kw = {}
        if tag == "zero":
            kw = dict(max_grad_norm=0.0, target_kl=0.0)
        elif tag == "null":                     # NULL options
            oc.with_null_options(m)
            kw = dict(max_grad_norm=0.0)
        elif tag == "stop":                     # a stop word and no guard
            kw = dict(stop=m.new_stop_word())
        mets = [m.train(s[idx], a[idx], ret[idx], adv[idx], **kw).cpu().numpy() for idx in np.split(perms[0][:768], 3)]
        out[tag] = (oc.model_state(m), np.stack(mets))
    for tag in ("zero", "null", "stop"):
        _same_state(out[tag][0], out["plain"][0])
        assert out[tag][1].shape == (3, 7) and np.array_equal(out[tag][1][:, :5], out["plain"][1])


# ------------------------------------------------------------------------------------------------ 2. clipping alone
def test_clipping_at_config3_matches_the_oracle(tmp_path):
    data = baseline_config3(oc.T3, oc.E3)
    max_norm = oc.pick_clip(data)
    m = oc.shipped_model(tmp_path / "clip")
    met = _learn(m, data, max_grad_norm=max_norm)
    rec64, n = _check_against_oracle(m, met, data, max_grad_norm=max_norm)
    clipped = rec64[:, 6] > max_norm
    assert clipped.mean() >= 0.25 and (~clipped).mean() >= 0.25, rec64[:, 6]
    assert n == oc.E3 * 8
    assert np.array_equal(m.adam_powers.cpu().numpy(), _powers_after(n))


# ------------------------------------------------------------------------------------------------ 3. KL stop
def test_kl_stop_mid_update_matches_the_oracle(tmp_path):
    data = baseline_config3(oc.T3, oc.E3)
    kl = oc.shipped_restate(data, np.float64, lr=oc.LR_KL)[2][:, 5]
    k, target = oc.pick_target(kl)
    thr = 1.5 * target
    assert kl[k] >= oc.MARGIN * thr and np.max(kl[:k]) * oc.MARGIN <= thr, (k, kl[:k + 1], thr)
    assert k > 1
    m = oc.shipped_model(tmp_path / "kl", lr=oc.LR_KL)
    met = _learn(m, data, target_kl=target)
    _, n = _check_against_oracle(m, met, data, target_kl=target, lr=oc.LR_KL)
    assert n == k and int(m.last_steps_applied.item()) == k
    assert np.array_equal(m.adam_powers.cpu().numpy(), _powers_after(k))          # advanced exactly k times
    assert not np.isnan(met[:k + 1]).any() and np.isnan(met[k + 1:]).all()      # the stopping row is written


def test_kl_stop_at_the_first_step_leaves_the_model_as_it_was(tmp_path):
    """train steps against ckpt-705's policy_old (a different old policy): the first step's approx_kl is far above a tiny
    target, so neither it nor the next step with the same stop word touches the model."""
    s, a, r, v, d, perms = baseline_config3(oc.T3, 1)
    rs = np.random.RandomState(3)
    ret, adv = rs.randn(oc.T3).astype(np.float32), rs.randn(oc.T3).astype(np.float32)
    m = oc.shipped_model(tmp_path / "first", lr=oc.LR_KL)
    before = oc.model_state(m)
    stop = m.new_stop_word()
    idx = np.split(perms[0][:512], 2)
    met0 = m.train(s[idx[0]], a[idx[0]], ret[idx[0]], adv[idx[0]], target_kl=1e-9, stop=stop).cpu().numpy()
    assert int(m.last_steps_applied.item()) == 0 and int(stop.item()) != 0
    assert met0[5] > 1.5e-9 and not np.isnan(met0).any()
    met1 = m.train(s[idx[1]], a[idx[1]], ret[idx[1]], adv[idx[1]], target_kl=1e-9, stop=stop).cpu().numpy()
    assert int(m.last_steps_applied.item()) == 0 and np.isnan(met1).all()
    _same_state(oc.model_state(m), before)


def test_a_target_that_never_triggers_is_the_clip_only_run(tmp_path):
    data = baseline_config3(oc.T3, oc.E3)
    runs = []
    for tag, kw in (("clip", dict(max_grad_norm=300.0)), ("both", dict(max_grad_norm=300.0, target_kl=1e3))):
        m = oc.shipped_model(tmp_path / tag, lr=oc.LR_KL)
        runs.append((_learn(m, data, **kw), m))
    (met_a, a), (met_b, b) = runs
    _same_state(oc.model_state(a), oc.model_state(b))
    assert np.array_equal(met_a, met_b) and int(b.last_steps_applied.item()) == oc.E3 * 8


# ------------------------------------------------------------------------------------------------ 4. both guards, segments
@pytest.mark.parametrize("lengths", [[128] * 16, [300, 1, 129, 700, 64, 854]], ids=["16x128", "ragged"])
def test_both_guards_over_segments_match_the_oracle(tmp_path, lengths):
    data = oc.segment_rollout(lengths, seed=len(lengths))
    rec = oc.shipped_restate(data, np.float64, lr=oc.LR_KL, lengths=lengths)[2]
    max_norm = float(np.median(rec[:, 6]))
    rec = oc.shipped_restate(data, np.float64, max_grad_norm=max_norm, lr=oc.LR_KL, lengths=lengths)[2]
    k, target = oc.pick_target(rec[:, 5])
    m = oc.shipped_model(tmp_path / "seg", lr=oc.LR_KL)
    met = _learn(m, data, lengths, max_grad_norm=max_norm, target_kl=target)
    _, n = _check_against_oracle(m, met, data, lengths=lengths, max_grad_norm=max_norm, target_kl=target,
                                 lr=oc.LR_KL)
    assert n == k


# ------------------------------------------------------------------------------------------------ 5. persistent, reference loop
def test_persistent_kernel_matches_launch_per_kernel(tmp_path):
    """CPB_PPO_PERSISTENT is read once per process: each path runs in a child process.  In each, the options twin with
    {0, 0} and NULL options is the original entry point bit for bit; across them the guarded update agrees at 1e-6 with
    the same number of applied steps."""
    data = baseline_config3(oc.T3, oc.E3)
    rec = oc.shipped_restate(data, np.float64, max_grad_norm=300.0, lr=oc.LR_KL)[2]
    k, target = oc.pick_target(rec[:, 5])
    ckpt = lambda null: ("ckpt705", oc.T3, oc.E3, oc.B3, "policy_old", oc.LR_KL, null)
    zero = dict(max_grad_norm=0.0, target_kl=0.0)
    outs = fresh_process(tmp_path, [("plain", REFERENCE, ckpt(False), {}), ("zero", REFERENCE, ckpt(False), zero),
                                    ("null", REFERENCE, ckpt(True), zero),
                                    ("guarded", REFERENCE, ckpt(False), dict(max_grad_norm=300.0, target_kl=target))],
                         timeout=600)
    for flag, z in zip("01", outs):
        for tag in ("zero", "null"):
            for key in KEYS:
                assert np.array_equal(z[tag + ":" + key], z["plain:" + key]), (flag, tag, key)
            assert np.array_equal(z[tag + ":metrics"][:, :5], z["plain:metrics"]), (flag, tag)
        assert int(z["guarded:applied"][0]) == k, flag
    for key in ("params", "m", "v"):
        assert rel_l2(outs[1]["guarded:" + key], outs[0]["guarded:" + key]) < 1e-6, key
    assert np.array_equal(outs[1]["guarded:powers"], outs[0]["guarded:powers"])
    assert np.array_equal(np.isnan(outs[1]["guarded:metrics"]), np.isnan(outs[0]["guarded:metrics"]))


def test_reference_loop_of_train_steps_is_learn(tmp_path):
    """The reference's Python loop over PPO.train (train.py --reference_loop) with one stop word per update stops where
    PPO.learn does and agrees with it at 1e-6."""
    from carla_ppo_b200.utils import compute_gae
    data = baseline_config3(oc.T3, oc.E3)
    s, a, r, v, d, perms = data
    rec = oc.shipped_restate(data, np.float64, max_grad_norm=300.0, lr=oc.LR_KL)[2]
    k, target = oc.pick_target(rec[:, 5])
    guards = dict(max_grad_norm=300.0, target_kl=target)
    ml = oc.shipped_model(tmp_path / "learn", lr=oc.LR_KL)
    met_l = _learn(ml, data, **guards)
    mt = oc.shipped_model(tmp_path / "loop", lr=oc.LR_KL)
    adv = compute_gae(list(r), list(v), 0.3, list(d), 0.99, 0.95)
    ret = adv + v
    adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    mt.update_old_policy()
    stop = mt.new_stop_word()
    applied, mets = 0, []
    for e in range(oc.E3):
        for i in range(oc.T3 // oc.B3):
            mb = perms[e][i * oc.B3:(i + 1) * oc.B3]
            mets.append(mt.train(s[mb], a[mb], ret[mb], adv[mb], stop=stop, **guards).cpu().numpy())
            applied += int(mt.last_steps_applied.item())
    assert applied == int(ml.last_steps_applied.item()) == k
    assert np.array_equal(np.isnan(np.stack(mets)), np.isnan(met_l))
    for key, x in oc.model_state(mt).items():
        assert rel_l2(x, oc.model_state(ml)[key]) < 1e-6, key


# ------------------------------------------------------------------------------------------------ 6. repeatability
def test_two_identical_calls_are_bit_identical(tmp_path):
    data = oc.segment_rollout(SEGMENTS, seed=5)
    runs = []
    for tag in ("a", "b"):
        m = oc.shipped_model(tmp_path / tag, lr=oc.LR_KL)
        met = _learn(m, data, SEGMENTS, max_grad_norm=100.0, target_kl=0.02)
        runs.append((oc.model_state(m), met, int(m.last_steps_applied.item())))
    _same_state(runs[0][0], runs[1][0])
    assert np.array_equal(runs[0][1], runs[1][1], equal_nan=True) and runs[0][2] == runs[1][2]


# ------------------------------------------------------------------------------------------------ 7. train.train
def test_train_with_four_environments_and_both_guards(tmp_path):
    """train.train --num_envs 4 --max_grad_norm 0.5 --target_kl 0.01: fused == unfused bit for bit."""
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    rgb, _ = committed_frames()
    models = []
    for tag, unfused in (("fused", False), ("unfused", True)):
        envs = [ReplayEnv(rgb, episode_length=24 + 5 * i, seed=0) for i in range(4)]
        params = train_params(tag, num_envs=4, max_grad_norm=0.5, target_kl=0.01, unfused=unfused)
        models.append(train(params, restart=False, env=envs, vae=shipped_vae(tmp_path, tag),
                            models_root=str(tmp_path / "models"), interactive=False))
    a, b = models
    assert a.last_steps_applied is not None and a.get_episode_idx() == 2
    _same_state(oc.model_state(a), oc.model_state(b))
    assert a.reward_history == b.reward_history
