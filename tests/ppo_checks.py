"""Checks that the PPO test modules share: the NaN-filled workspace, the float32-distance gate, the loss / Adam-step /
learn checks against tests/ppo_restatement.py, the actor VAEs and fake environments, learn() in a fresh process per
CPB_PPO_PERSISTENT setting, and the table of every cpb_ppo_* entry point with arguments that are refused before any
launch."""
import ctypes as C
import os
import pickle
import subprocess
import sys
import types

import numpy as np

import ppo_restatement as pr
from helpers import committed_frames, rel_l2

TOL = 1e-5
METRICS = ("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio")


# ------------------------------------------------------------------------------------------------------------ gates
def nan_workspace(m, *shape):
    ws = m._workspace(*shape)
    ws.fill_(0xFF)                  # every float of the workspace reads as NaN until written
    return ws


def gate(got, r64, r32):
    """max(TOL, 2 x the float32 restatement's distance from float64)"""
    return rel_l2(got, r64) < max(TOL, 2 * rel_l2(r32, r64))


def check_loss(m, p, old, s, a, ret, adv, head, entropy_scale=0.01):
    """PPO.loss_and_grads against the restatement in float64, gated by float32's distance; a loss term that is exactly 0
    in float64 (no entropy, no advantage) must be exactly 0.  -> the float64 result"""
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    r64 = pr.loss_and_grads(p, old, s, a, ret, adv, head, 0.2, 1.0, entropy_scale)
    r32 = pr.loss_and_grads(p, old, s, a, ret, adv, head, 0.2, 1.0, entropy_scale, dtype=np.float32)
    assert np.isfinite(metrics).all()
    for i, k in enumerate(METRICS):
        if r64[k] == 0.0:
            assert metrics[i] == 0.0, k
            continue
        assert gate(np.atleast_1d(metrics[i]), np.atleast_1d(r64[k]), np.atleast_1d(r32[k])), k
    assert set(grads) == set(r64["grads"])
    for k, g in grads.items():
        assert np.isfinite(g).all(), k
        assert gate(g, r64["grads"][k], r32["grads"][k]), (k, rel_l2(g, r64["grads"][k]))
    return r64


def check_two_train_steps(tmp_path, net, batch):
    """Two PPO.train steps from warm Adam slots against two restated Adam steps."""
    from oracle import vae_oracle as vo
    from ppo_cases import LR, make_ppo, warm_adam
    head = net[1]
    p, old, s, a, ret, adv = batch
    m_, v_, powers = warm_adam(p, pr.loss_and_grads(p, old, s, a, ret, adv, head, 0.2, 1.0, 0.01)["grads"], 19)
    m = make_ppo(tmp_path, net, p, old)
    m.set_weights(p, old, m_, v_, powers)
    for _ in range(2):
        nan_workspace(m, len(s))
        m.train(s, a, ret, adv)

    def steps(dtype):
        q = {k: x.astype(dtype) for k, x in p.items()}
        st = dict(m={k: m_[k].astype(dtype) for k in p}, v={k: v_[k].astype(dtype) for k in p}, beta1_power=powers[0],
                  beta2_power=powers[1])
        for _ in range(2):
            vo.adam_apply(q, pr.loss_and_grads(q, old, s, a, ret, adv, head, 0.2, 1.0, 0.01, dtype=dtype)["grads"], st, LR)
        return q
    p64, p32 = steps(np.float64), steps(np.float32)
    got = m.get_weights()
    for k in p64:
        assert gate(got[k], p64[k], p32[k]), k


def five(refs):
    """learn_refs with the records cut to the five losses (no guards: the device reports five columns)"""
    return (refs[0][0], refs[0][1][:, :5], refs[0][2]), (refs[1][0], refs[1][1][:, :5], 0)


def check_learn(got, metrics, refs, applied=None):
    """Weights and metric rows of a learn() against learn_refs: the same NaN rows (a KL stop), every evaluated row
    within the gate (approx_kl, column 5, is 0 at the first minibatch and ~1e-8 soon after: gated absolutely as well),
    and the Adam steps applied."""
    (p64, rec64, n64), (p32, rec32, _) = refs
    for k in p64:
        assert np.isfinite(got[k]).all(), k
        assert gate(got[k], p64[k], p32[k]), (k, rel_l2(got[k], p64[k]))
    ok = ~np.isnan(rec64[:, 0])
    assert np.array_equal(np.isnan(metrics[:, 0]), ~ok)
    for col in range(metrics.shape[1]):
        assert (gate(metrics[ok, col], rec64[ok, col], rec32[ok, col])
                or (col == 5 and np.abs(metrics[ok, col] - rec64[ok, col]).max() < 1e-6)), col
    if applied is not None:
        assert applied == n64


def check_learn_segments(tmp_path, net):
    """learn() over 16 segments x 128 rows, 2 epochs of minibatches of 256."""
    from ppo_cases import learn_refs, learn_setup, make_ppo
    p, data, perms, adam = learn_setup(net, 2048, 2, 50)
    s, a, r, v, d = data
    lengths = [128] * 16
    boot = np.random.RandomState(51).randn(16)
    m = make_ppo(tmp_path, net, p)
    m.set_weights(p, p, *adam)
    nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, boot, num_epochs=2, batch_size=256, perms=perms, return_metrics=True,
                      segment_lengths=lengths)
    check_learn(m.get_weights(), metrics, five(learn_refs(net, p, data, perms, 256, adam, segment_lengths=lengths,
                                                          bootstrap_values=boot)))


def check_learn_opts_clip_and_kl_stop(tmp_path, net):
    """Clipping binding on 25-75 % of the minibatches, then a KL stop at a minibatch k > 1 (steps_applied = k).  The
    learning rate is 3e-3 so that the approximate KL of the later minibatches stands well above float32 rounding."""
    from ppo_cases import learn_refs, learn_setup, make_ppo
    lr = 3e-3
    p, data, perms, adam = learn_setup(net, 2048, 4, 60)
    s, a, r, v, d = data
    # the pre-clip norms of the unguarded update set the clip; its KL values set the stop
    (_, rec0, _), _ = learn_refs(net, p, data, perms, 256, adam, lr=lr)
    for q in (0.375, 0.5, 0.625):          # the first quantile of the unclipped norms that clips 25-75 % of the steps
        max_norm = float(np.quantile(rec0[:, 6], q))
        (_, rec, _), _ = learn_refs(net, p, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm)
        clipped = (rec[:, 6] > max_norm).mean()
        if 0.25 <= clipped <= 0.75:
            break
    assert 0.25 <= clipped <= 0.75, clipped
    kl = rec[:, 5]
    # the first minibatch from the third on whose KL exceeds every earlier one by 20 %, and is above float32 noise
    k = next(i for i in range(2, len(kl)) if kl[i] > 1.2 * kl[:i].max() and kl[i] > 1e-5)
    target_kl = float((kl[:k].max() + kl[k]) / 2 / 1.5)
    refs = learn_refs(net, p, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm, target_kl=target_kl)
    assert refs[0][2] == k > 1, (refs[0][2], k)
    m = make_ppo(tmp_path, net, p, learning_rate=lr)
    m.set_weights(p, p, *adam)
    nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=4, batch_size=256, perms=perms, return_metrics=True,
                      max_grad_norm=max_norm, target_kl=target_kl)
    check_learn(m.get_weights(), metrics, refs, applied=int(m.last_steps_applied.item()))


def torch_loss_and_grads(p, old, s, a, ret, adv, head, epsilon=0.2, value_scale=1.0, entropy_scale=0.01):
    """The PPO loss of either head written out in torch float64 from the spec, not from the restatement, with autograd
    for the gradients.  -> (loss, {name: gradient})"""
    import torch
    from oracle import ppo_oracle as po
    t = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in p.items()}
    o = {k: torch.tensor(np.asarray(v, np.float64)) for k, v in old.items()}
    x = torch.tensor(np.asarray(s, np.float64))
    pol, val = pr.trunk_names(p)

    def trunk(q, layers):
        h = x
        for w, b in layers:
            h = torch.relu(h @ q[w] + q[b])
        return h
    if pr.is_categorical(head):
        off, ai = pr.offsets(head), torch.tensor(np.asarray(a).astype(np.int64))

        def logp_and_h(q):
            z = trunk(q, pol) @ q["action_logits/kernel"] + q["action_logits/bias"]
            lp, H = 0.0, 0.0
            for k in range(len(head)):
                l = torch.log_softmax(z[:, off[k]:off[k + 1]], dim=1)
                lp = lp + l.gather(1, ai[:, k:k + 1])[:, 0]
                H = H - (l.exp() * l).sum(dim=1)
            return lp, H
        (lp, H), (lp_old, _) = logp_and_h(t), logp_and_h(o)
        advt, entropy = torch.tensor(np.asarray(adv, np.float64)), H.mean()
    else:
        lo, hi, act = torch.tensor(head[0]), torch.tensor(head[1]), torch.tensor(np.asarray(a, np.float64))

        def logp(q):
            mu = lo + (torch.tanh(trunk(q, pol) @ q["action_mean/kernel"] + q["action_mean/bias"]) + 1) / 2 * (hi - lo)
            ls = q["action_logstd"]
            return (-0.5 * ((act - mu) / torch.exp(ls)) ** 2 - (po.LOG_SQRT_2PI + ls)).sum(-1, keepdim=True)
        lp, lp_old = logp(t), logp(o)
        advt, entropy = torch.tensor(np.asarray(adv, np.float64))[:, None], torch.sum(po.ENTROPY_CONST + t["action_logstd"])
    v = (trunk(t, val) @ t["value/kernel"] + t["value/bias"])[:, 0]
    ratio = torch.exp(lp - lp_old)
    clo, chi = float(np.float32(1 - epsilon)), float(np.float32(1 + epsilon))
    pl = torch.mean(torch.minimum(ratio * advt, torch.clamp(ratio, clo, chi) * advt))
    vl = torch.mean((v - torch.tensor(np.asarray(ret, np.float64))) ** 2) * float(np.float32(value_scale))
    loss = -pl + vl - entropy * float(np.float32(entropy_scale))
    loss.backward()
    return float(loss.detach()), {k: g.grad.numpy() for k, g in t.items()}


# ------------------------------------------------------------------------------------------------------ fused actor
def actor_vae(tmp_path, kind):
    from harness import make_conv_vae, make_mlp
    from helpers import shipped_vae_weights
    from vae_checks import mlp_weights
    if kind == "conv":
        return make_conv_vae(tmp_path, shipped_vae_weights()[0], loss="bce", tag="vae", training=False)
    enc, dec = (96, 256, 64), (160, 64)
    return make_mlp(tmp_path, mlp_weights(2, encoder_sizes=enc, decoder_sizes=dec), enc, dec, tag="vec", training=False)


def check_fused_actor(tmp_path, net, kind, n, greedy):
    """FusedActor.encode_predict bit for bit UnfusedActor's at `net` for each of the `greedy` settings: states, actions
    and values (a categorical policy far from uniform: int64 indices in range)."""
    from carla_ppo_b200.actor import FusedActor, UnfusedActor
    from ppo_cases import make_ppo
    head = net[1]
    vae = actor_vae(tmp_path, kind)
    meas = ("steer", "throttle", "speed")
    p = pr.init_params(*net, seed=90)
    if pr.is_categorical(head):
        p["action_logits/bias"] = np.random.RandomState(91).randn(sum(head)).astype(np.float32)
    models = [make_ppo(tmp_path / tag, net, p) for tag in ("fused", "unfused")]
    envs = fake_envs(n)
    for g in greedy:
        fa_, ua_ = FusedActor(vae, models[0], meas), UnfusedActor(vae, models[1], meas)
        fa_.greedy = ua_.greedy = g
        fs, fa, fv = fa_.encode_predict(envs)
        us, ua, uv = ua_.encode_predict(envs)
        assert all(np.array_equal(x, y) for x, y in zip(fs, us))
        assert np.array_equal(fa, ua) and np.array_equal(fv, uv)
        if pr.is_categorical(head):
            assert fa.dtype == ua.dtype == np.int64
            assert (fa >= 0).all() and (fa < np.asarray(head)).all()
        else:
            assert np.isfinite(fa).all()


def fake_envs(n):
    rgb, _ = committed_frames()
    envs = []
    for i in range(n):
        v = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.1 * (i % 7) - 0.3, throttle=0.05 * (i % 11)),
                                  get_speed=(lambda s=0.37 * i: s))
        envs.append(types.SimpleNamespace(observation=rgb[(5 * i) % len(rgb)], vehicle=v))
    return envs


# ------------------------------------------------------------------------------------------------ a fresh process
def fresh_process(tmp_path, cases, flags=("0", "1"), body="learn_cases", timeout=1200):
    """body(model_dir, cases, out) of this module in a fresh Python process per CPB_PPO_PERSISTENT flag (the variable is
    read once per process).  -> one dict of the arrays body saved per flag"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(tmp_path / "cases.pkl", "wb") as f:
        pickle.dump(cases, f)
    outs = []
    for flag in flags:
        out = str(tmp_path / ("out%s.npz" % flag))
        code = ("import sys, pickle; sys.path[:0] = [%r, %r]; import ppo_checks; "
                "ppo_checks.%s(%r, pickle.load(open(%r, 'rb')), %r)"
                % (root, os.path.join(root, "tests"), body, str(tmp_path / ("m" + flag)), str(tmp_path / "cases.pkl"),
                   out))
        res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_PPO_PERSISTENT=flag),
                             capture_output=True, text=True, timeout=timeout)
        assert res.returncode == 0, res.stderr[-3000:]
        outs.append(dict(np.load(out)))
    return outs


def learn_cases(model_dir, cases, out):
    """Child side of fresh_process: one learn() per case (tag, net, setup, learn keyword arguments) from a fresh PPO.
    setup = ("rollout", T, epochs, batch, seed): ppo_cases.learn_setup's rollout, weights and warm Adam slots, with the
    workspace filled with NaN; or ("ckpt705", T, epochs, batch, old, lr, null_options): ckpt-705's policy, `old` as
    theta_old ("policy" or "policy_old") and its Adam state over baseline_config3(T, epochs).  Saves, per tag, every
    weight ("w:" + name), the flat state (params, old, m, v, powers), the metrics and steps_applied."""
    from pathlib import Path
    import ppo_cases as pc
    from helpers import shipped_ppo
    res = {}
    for tag, net, setup, kw in cases:
        kind, T, epochs, batch = setup[:4]
        if kind == "rollout":
            p, (s, a, r, v, d), perms, adam = pc.learn_setup(net, T, epochs, setup[4])
            m = pc.make_ppo(Path(model_dir) / tag, net, p)
            m.set_weights(p, p, *adam)
            nan_workspace(m, min(batch, T), T)
            last = 0.3
        else:
            old_prefix, lr, null_options = setup[4:]
            pol, _ = shipped_ppo("policy")
            m = pc.make_ppo(Path(model_dir) / tag, net, pol, learning_rate=lr)
            m.set_weights(pol, shipped_ppo(old_prefix)[0], *pc.shipped_adam())
            if null_options:
                pc.with_null_options(m)
            s, a, r, v, d, perms = pc.baseline_config3(T, epochs)
            last = 0.3 if kw.get("segment_lengths") is None else [0.3]
        res[tag + ":metrics"] = m.learn(s, a, v, r, d, last, num_epochs=epochs, batch_size=batch, perms=perms,
                                        return_metrics=True, **kw)
        res.update({tag + ":w:" + k: x for k, x in m.get_weights().items()})
        res.update({tag + ":" + k: x for k, x in pc.model_state(m).items()})
        if m.last_steps_applied is not None:
            res[tag + ":applied"] = m.last_steps_applied.cpu().numpy()
    np.savez(out, **res)


def spec_vs_legacy(model_dir, seed, out):
    """Child side of the default-architecture test: learn, learn_opts, learn_segments and learn_segments_opts through
    the spec twins (use_spec 1) and through the legacy entry points, the spec names mapped back (use_spec 0)."""
    from pathlib import Path
    import ppo_cases as pc
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    net = pc.gauss_net(pc.ARCHS["default"])
    p, data, perms, adam = pc.learn_setup(net, 2048, 2, seed)
    s, a, r, v, d = data
    res = {}
    for use_spec in (0, 1):
        m = pc.make_ppo(Path(model_dir) / str(use_spec), net, p)
        if not use_spec:
            real = m._call
            m._call = lambda name, *args, _r=real, _m=m: _r(name.replace("cpb_ppo_spec_", "cpb_ppo_"),
                                                            *((C.byref(_m._c),) + args[1:]))
        for opts in ({}, {"max_grad_norm": 0.05, "target_kl": 0.004}):
            for seg in (None, [1024, 1024]):
                m.set_weights(p, p, *adam)
                lib.cpb_reset_launch_count()
                boot = 0.3 if seg is None else np.array([0.3, -0.1])
                met = m.learn(s, a, v, r, d, boot, num_epochs=2, batch_size=256, perms=perms, return_metrics=True,
                              segment_lengths=seg, **opts)
                tag = "%d:%d:%d" % (use_spec, bool(opts), seg is not None)
                res[tag + ":launches"] = np.int64(lib.cpb_launch_count())
                res[tag + ":metrics"] = met
                res.update({tag + ":" + k: x for k, x in pc.model_state(m).items()})
                if opts:
                    res[tag + ":applied"] = m.last_steps_applied.cpu().numpy()
    np.savez(out, **res)


# ------------------------------------------------------------------------------------------------ refused calls
FAKE = 1 << 44          # never dereferenced: every call made with these arguments must be refused before any launch
WS_BYTES = 1 << 40      # large enough for any plan; the pointer is never used
STEP_POINTERS = ("params", "params_old", "grads", "adam_m", "adam_v", "adam_powers", "lr_dev", "states", "actions",
                 "returns", "advantages")
LEARN_POINTERS = STEP_POINTERS[:9] + ("rewards", "values", "dones", "perms")
SEGMENTS_POINTERS = STEP_POINTERS[:9] + ("rewards", "values", "bootstrap", "dones", "offsets", "perms")
# entry point -> arguments after the descriptor, from a dict `a` of pointers and sizes (ppo_args fills the defaults)
_STEP = lambda a: tuple(a[k] for k in STEP_POINTERS) + (None, a["B"], FAKE)
_LEARN = lambda a: (tuple(a[k] for k in LEARN_POINTERS[:11])
                    + (0.3, a["dones"], a["rows"], 0.99, 0.95, a["epochs"], a["batch"], a["perms"], FAKE))
_SEGMENTS = lambda a: (tuple(a[k] for k in SEGMENTS_POINTERS[:14])
                       + (a["S"], a["rows"], 0.99, 0.95, a["epochs"], a["batch"], a["perms"], FAKE))
_WS = lambda a: (a["ws"], a["ws_bytes"], None)
ARGS = {
    "num_tensors": lambda a: (),
    "layout": lambda a: (None, None, None, None),
    "workspace_bytes": lambda a: (4, 0),
    "forward": lambda a: (a["params"], a["states"], a["B"], None, FAKE, FAKE) + _WS(a),
    "loss_grad": lambda a: (a["params"], a["params_old"], a["states"], a["actions"], a["returns"], a["advantages"], None,
                            a["B"], a["grads"], FAKE) + _WS(a),
    "train_step": lambda a: _STEP(a) + _WS(a),
    "train_step_opts": lambda a: _STEP(a) + (a["opts"], FAKE, FAKE) + _WS(a),
    "learn": lambda a: _LEARN(a) + _WS(a),
    "learn_opts": lambda a: _LEARN(a) + (a["opts"], FAKE) + _WS(a),
    "learn_segments": lambda a: _SEGMENTS(a) + _WS(a),
    "learn_segments_opts": lambda a: _SEGMENTS(a) + (a["opts"], FAKE) + _WS(a),
    "vae_actor": lambda a: (FAKE, FAKE, FAKE, 3, a["desc"], FAKE, None, FAKE, FAKE, FAKE, FAKE, None, a["ws"],
                            a["ws_bytes"], a["ws"], a["ws_bytes"], None),
    "mlp_actor": lambda a: (FAKE, FAKE, FAKE, 3, a["desc"], FAKE, None, FAKE, FAKE, FAKE, FAKE, None, a["ws"],
                            a["ws_bytes"], a["ws"], a["ws_bytes"], None),
}
SPEC_ENTRIES = list(ARGS)
LEGACY_OPTS_ENTRIES = {"learn_opts": LEARN_POINTERS, "learn_segments_opts": SEGMENTS_POINTERS,
                       "train_step_opts": STEP_POINTERS}


def entry_name(family, entry):
    """family "cpb_ppo_", "cpb_ppo_spec_" or "cpb_ppo_cat_": its C entry point for `entry` (an ARGS key)"""
    if entry.endswith("actor"):
        return ("cpb_vae_spec_ppo_%sencode_predict" if entry == "vae_actor" else "cpb_mlpvae_ppo_%sencode_predict") \
            % family[len("cpb_ppo_"):]
    return family + entry


def ppo_args(entry, desc, opts=None, **over):
    """The arguments of `entry` with the descriptor `desc` (a ctypes reference or None), FAKE pointers, 40 rows in
    S = 3 segments, 2 epochs of minibatches of 16, train steps of 16 rows; `over` replaces any pointer or size."""
    from carla_ppo_b200 import _lib
    a = {k: FAKE for k in SEGMENTS_POINTERS + STEP_POINTERS}
    a.update(desc=desc, opts=opts, B=16, rows=40, S=3, epochs=2, batch=16, ws=FAKE, ws_bytes=WS_BYTES)
    if entry.endswith("actor"):
        cfg = _lib.VaeConfig(4, 3, 64, 1, 1, 0, 1.0, 1.0, 0.0, 1.0)
        a.update(vae=C.byref(_lib.VaeSpec(cfg, 80, 160)), mlp=C.byref(_lib.MlpVaeSpec.of(cfg, (512, 256), (256, 512))))
    a.update(over)
    return ({"vae_actor": a.get("vae"), "mlp_actor": a.get("mlp")}.get(entry, desc),) + ARGS[entry](a)


def ppo_call(lib, family, entry, desc, opts=None, **over):
    return getattr(lib, entry_name(family, entry))(*ppo_args(entry, desc, opts, **over))
