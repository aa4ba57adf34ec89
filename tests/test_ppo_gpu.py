"""GPU parity tests of the PPO update path (C ABI through the reference-shaped PPO class) against the
float64 oracle.  Tolerance: ||x - ref|| / ||ref|| <= 1e-5 for forward quantities, losses and updated
parameters; gradients <= max(2 x fp32-CPU-restatement error, 2e-5) per tensor."""
import numpy as np
import pytest

from helpers import rel_l2, shipped_ppo
from ppo_cases import HIGH, LOW, REFERENCE, baseline_config3, make_ppo
from ppo_checks import fresh_process

pytestmark = pytest.mark.gpu

TOL = 1e-5


def rollout(T, seed=0):
    rs = np.random.RandomState(seed)
    states = rs.randn(T, 67).astype(np.float32)
    actions = np.clip(rs.randn(T, 2), LOW, HIGH).astype(np.float32)
    rewards = rs.rand(T)
    values = rs.randn(T).astype(np.float32)
    dones = np.zeros(T, bool); dones[-1] = True
    return states, actions, rewards, values, dones


def test_predict_matches_oracle(tmp_path):
    from oracle import ppo_oracle as po
    pol, _ = shipped_ppo("policy")
    m = make_ppo(tmp_path, REFERENCE, pol)
    states = rollout(33)[0]
    p64 = {k: v.astype(np.float64) for k, v in pol.items()}
    act, val = m.predict(states, greedy=True)
    ract, rval = po.predict(p64, states, LOW, HIGH)
    assert act.shape == (33, 2) and val.shape == (33,)
    assert rel_l2(act, ract) < TOL and rel_l2(val, rval) < TOL
    noise = np.random.RandomState(5).randn(33, 2)
    act, _ = m.predict(states, noise=noise)
    ract, _ = po.predict(p64, states, LOW, HIGH, noise=noise)
    assert rel_l2(act, ract) < TOL
    assert (act >= LOW - 1e-7).all() and (act <= HIGH + 1e-7).all()
    a1, v1 = m.predict(states[0], greedy=True)              # B=1 squeeze (ppo.py:249-250)
    assert a1.shape == (2,) and np.ndim(v1) == 0
    assert rel_l2(a1, ract[0] * 0 + po.predict(p64, states[0], LOW, HIGH)[0]) < TOL


@pytest.mark.parametrize("batch", [256, 37])
def test_loss_and_gradients_match_oracle(tmp_path, batch):
    import torch
    from oracle import ppo_oracle as po, torch_ref
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = make_ppo(tmp_path, REFERENCE, pol, old)
    rs = np.random.RandomState(1)
    s, a = rollout(batch, 2)[:2]
    ret = rs.randn(batch).astype(np.float32); adv = rs.randn(batch).astype(np.float32)
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    ref = po.loss_and_grads(pol, old, s, a, ret, adv, LOW, HIGH, 0.2, 1.0, 0.01)
    ref32 = torch_ref.ppo_loss_and_grads(pol, old, s, a, ret, adv, LOW, HIGH, 0.2, 1.0, 0.01, dtype=torch.float32)
    for got, key in zip(metrics, ("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio")):
        assert abs(got - ref[key]) <= TOL * max(abs(ref[key]), 1e-3), key
    for name, g in ref["grads"].items():
        err = rel_l2(grads[name], g)
        tol = max(2 * rel_l2(ref32["grads"][name], g), 2e-5)
        assert err < tol, "%s: %.3e (fp32 cpu %.3e)" % (name, err, tol / 2)


def test_train_step_matches_oracle(tmp_path):
    from oracle import ppo_oracle as po, vae_oracle as vo
    pol, z = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = make_ppo(tmp_path, REFERENCE, pol, old)
    s, a = rollout(64, 3)[:2]
    rs = np.random.RandomState(4)
    ret = rs.randn(64).astype(np.float32); adv = rs.randn(64).astype(np.float32)
    p64 = {k: v.astype(np.float64) for k, v in pol.items()}
    st = vo.adam_init_state(p64)
    for _ in range(2):
        m.train(s, a, ret, adv)
        out = po.loss_and_grads(p64, old, s, a, ret, adv, LOW, HIGH, 0.2, 1.0, 0.01)
        vo.adam_apply(p64, out["grads"], st, 1e-4)
    got = m.get_weights()
    for name in p64:
        assert rel_l2(got[name], p64[name]) < TOL, name
    assert m.get_train_step_idx() == 2


def test_compute_gae_matches_reference_expression():
    from carla_ppo_b200.utils import compute_gae
    from oracle import ppo_oracle as po
    rs = np.random.RandomState(0)
    for T in (1, 5, 128, 2048, 2500):
        r = rs.rand(T); v = rs.randn(T); d = rs.rand(T) < 0.05
        got = compute_gae(list(r), list(v), 0.3, list(d), 0.99, 0.95)
        ref = po.compute_gae(r, v, 0.3, d, 0.99, 0.95)
        assert got.dtype == np.float64 and got.shape == (T,)
        assert rel_l2(got, ref) < 1e-12, T


def test_learn_matches_oracle_driver_block(tmp_path):
    """BASELINE config 3 shape at reduced size for the oracle: T=512, 2 epochs x minibatch 96 (short tail),
    shipped ckpt-705 weights; parameters after learn() vs the float64 restatement of train.py:171-207."""
    from oracle import ppo_oracle as po, vae_oracle as vo
    pol, _ = shipped_ppo("policy")
    m = make_ppo(tmp_path, REFERENCE, pol)
    T, E, B = 512, 2, 96
    s, a, r, v, d = rollout(T, 7)
    perms = np.stack([np.random.RandomState(10 + e).permutation(T) for e in range(E)])
    metrics = m.learn(s, a, v, r, d, 0.3, gamma=0.99, lam=0.95, num_epochs=E, batch_size=B, perms=perms, return_metrics=True)
    p64 = {k: x.astype(np.float64) for k, x in pol.items()}
    st = vo.adam_init_state(p64)
    rec = po.learn(p64, st, s, a, v, r, d, 0.3, LOW, HIGH, 0.99, 0.95, 1e-4, 0.2, 1.0, 0.01, E, B, perms)
    got = m.get_weights()
    for name in p64:
        assert rel_l2(got[name], p64[name]) < TOL, name
    rec = np.asarray(rec)
    assert metrics.shape == rec.shape
    assert np.allclose(metrics[:, 3], rec[:, 3], rtol=2e-4, atol=1e-5)      # total loss of every minibatch
    old = m.get_old_weights()
    assert all(np.array_equal(old[k], pol[k]) for k in pol)                 # theta_old == theta at learn() entry
    assert m.get_train_step_idx() == E * 6


def test_checkpoint_round_trip_and_lr_decay(tmp_path):
    pol, _ = shipped_ppo("policy")
    m = make_ppo(tmp_path, REFERENCE, pol, lr_decay=0.5)
    assert abs(float(m.learning_rate) - 1e-4) < 1e-11          # float32(1e-4), like the TF tensor
    m.write_episodic_summaries()
    assert m.get_episode_idx() == 1 and abs(float(m._lr_dev.item()) - 5e-5) < 1e-10
    m.save()
    m2 = make_ppo(tmp_path)
    assert m2.load_latest_checkpoint() is True
    assert m2.get_episode_idx() == 1
    w1, w2 = m.get_weights(), m2.get_weights()
    assert all(np.array_equal(w1[k], w2[k]) for k in w1)


def test_learn_at_baseline_config3_matches_oracle(tmp_path):
    """The driver's update block (reference train.py:171-207) at EXACTLY BASELINE configs[2]: parameters, theta_old and
    the 32 per-minibatch losses vs the float64 restatement; gate = max(1e-5, 2 x the error of the float32 CPU
    restatement run through the same 32 Adam steps)."""
    from oracle import ppo_oracle as po
    pol, z = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    adam_m = {k: z["adam_m/" + k] for k in pol}
    adam_v = {k: z["adam_v/" + k] for k in pol}
    powers = (float(z["beta1_power"]), float(z["beta2_power"]))
    m = make_ppo(tmp_path, REFERENCE, pol, old)
    m.set_weights(pol, old, adam_m, adam_v, powers)
    T, E, B = 2048, 4, 256
    s, a, r, v, d, perms = baseline_config3(T, E)
    metrics = m.learn(s, a, v, r, d, 0.3, gamma=0.99, lam=0.95, num_epochs=E, batch_size=B, perms=perms, return_metrics=True)

    def restate(dtype):
        p = {k: x.astype(dtype) for k, x in pol.items()}
        st = dict(m={k: adam_m[k].astype(dtype) for k in pol}, v={k: adam_v[k].astype(dtype) for k in pol},
                  beta1_power=powers[0], beta2_power=powers[1])
        rec = po.learn(p, st, s, a, v, r, d, 0.3, LOW, HIGH, 0.99, 0.95, 1e-4, 0.2, 1.0, 0.01, E, B, perms, dtype=dtype)
        return p, np.asarray(rec, np.float64)
    p64, rec64 = restate(np.float64)
    p32, rec32 = restate(np.float32)
    got = m.get_weights()
    for name in p64:
        gate = max(TOL, 2 * rel_l2(p32[name], p64[name]))
        assert rel_l2(got[name], p64[name]) < gate, "%s: %.3e (gate %.3e)" % (name, rel_l2(got[name], p64[name]), gate)
    assert metrics.shape == rec64.shape == (E * (T // B), 5)
    for col in range(5):
        gate = max(TOL, 2 * rel_l2(rec32[:, col], rec64[:, col]))
        assert rel_l2(metrics[:, col], rec64[:, col]) < gate, (col, rel_l2(metrics[:, col], rec64[:, col]), gate)
    gold = m.get_old_weights()
    assert all(np.array_equal(gold[k], pol[k]) for k in pol)               # update_old_policy() ran at entry
    assert m.get_train_step_idx() == 32


def test_update_old_policy_and_zero_epoch_learn(tmp_path):
    """PPO.update_old_policy (ppo.py:275-276) called directly; learn(num_epochs=0) still does theta_old <- theta."""
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = make_ppo(tmp_path, REFERENCE, pol, old)
    assert not all(np.array_equal(m.get_old_weights()[k], pol[k]) for k in pol)
    m.update_old_policy()
    assert all(np.array_equal(m.get_old_weights()[k], pol[k]) for k in pol)
    m.set_weights(pol, old)
    s, a, r, v, d = rollout(40, 3)
    out = m.learn(s, a, v, r, d, 0.1, num_epochs=0, batch_size=16, return_metrics=True)
    assert out.shape == (0, 5)
    assert all(np.array_equal(m.get_old_weights()[k], pol[k]) for k in pol)
    assert all(np.array_equal(m.get_weights()[k], pol[k]) for k in pol)


def test_persistent_learn_kernel_matches_launch_per_kernel_path(tmp_path):
    """CPB_PPO_PERSISTENT=1 (one cooperative kernel for all minibatch steps) vs the default launch-per-kernel learn():
    same parameters to fp32 round-off (the per-CTA loss partials are summed in a different order)."""
    # ragged last minibatch (2048 = 10 x 200 + 48)
    outs = fresh_process(tmp_path, [("ckpt", REFERENCE, ("ckpt705", 2048, 2, 200, "policy", 1e-4, False), {})])
    for k in shipped_ppo("policy")[0]:
        w0, w1 = outs[0]["ckpt:w:" + k], outs[1]["ckpt:w:" + k]
        assert rel_l2(w1, w0) < 1e-6, (k, rel_l2(w1, w0))
