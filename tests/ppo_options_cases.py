"""The cases the bounded-update GPU tests share: the reference agent at BASELINE configs[2] (ckpt-705 with its Adam state,
T = 2048, 4 epochs x 256), the float64 / float32 restatements of a guarded update there, the choice of a KL target that
stops the update at a known minibatch, and the run the persistent-kernel test makes in a child process."""
import numpy as np

import ppo_options_oracle as oo
from helpers import shipped_ppo
from ppo_cases import HIGH, LOW, baseline_config3, make_ppo

T, E, B = 2048, 4, 256
LR_KL = 1e-3          # large enough that the approximate KL grows from minibatch to minibatch (to ~1e-2)
MARGIN = 1.05         # both sides of a KL crossing stay this far from the stop threshold


def adam_state():
    pol, z = shipped_ppo("policy")
    return ({k: z["adam_m/" + k] for k in pol}, {k: z["adam_v/" + k] for k in pol},
            (float(z["beta1_power"]), float(z["beta2_power"])))


def model(path, lr=1e-4):
    """The PPO class at ckpt-705: policy, policy_old, warm Adam slots and beta powers."""
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = make_ppo(path, pol, old, learning_rate=lr)
    am, av, powers = adam_state()
    m.set_weights(pol, old, am, av, powers)
    return m


def state(m):
    return dict(params=m.params.cpu().numpy(), old=m.params_old.cpu().numpy(), m=m.adam_m.cpu().numpy(),
                v=m.adam_v.cpu().numpy(), powers=m.adam_powers.cpu().numpy())


def segment_rollout(lengths, seed=0):
    """configs[2]-shaped rows over segments: states, actions, rewards, values, dones, bootstrap values, perms."""
    from ppo_cases import segment_inputs
    rows = int(np.sum(lengths))
    rs = np.random.RandomState(seed)
    s = rs.randn(rows, 67).astype(np.float32)
    a = np.clip(rs.randn(rows, 2), LOW, HIGH).astype(np.float32)
    r, v, boot, d = segment_inputs(lengths, seed)
    perms = np.stack([np.random.RandomState(seed + 1 + e).permutation(rows) for e in range(E)])
    return s, a, r, v.astype(np.float32), d, boot, perms


def restate(data, dtype, max_grad_norm=0.0, target_kl=0.0, lr=1e-4, lengths=None):
    """The guarded update from ckpt-705 in `dtype`: (params, adam state, records [steps][7], steps applied).  data =
    baseline_config3's (s, a, r, v, d, perms), or segment_rollout's (s, a, r, v, d, boot, perms) with `lengths`."""
    pol, _ = shipped_ppo("policy")
    am, av, powers = adam_state()
    p = {k: x.astype(dtype) for k, x in pol.items()}
    st = dict(m={k: am[k].astype(dtype) for k in pol}, v={k: av[k].astype(dtype) for k in pol},
              beta1_power=powers[0], beta2_power=powers[1])
    if lengths is None:
        s, a, r, v, d, perms = data
        boot = None
    else:
        s, a, r, v, d, boot, perms = data
    rec, applied = oo.learn(p, st, s, a, v, r, d, 0.3, LOW, HIGH, 0.99, 0.95, lr, 0.2, 1.0, 0.01, E, B, perms, dtype,
                            max_grad_norm, target_kl, lengths, boot)
    return p, st, rec, applied


def pick_clip(data, lr=1e-4, lengths=None):
    """A max_grad_norm at which between a quarter and three quarters of the clipped update's minibatches clip: a multiple
    of the median pre-clip norm of the unclipped update (clipping slows the update, so its norms stay higher)."""
    base = float(np.median(restate(data, np.float64, lr=lr, lengths=lengths)[2][:, 6]))
    for f in (1.0, 1.5, 2.0, 3.0, 4.0):
        norms = restate(data, np.float64, max_grad_norm=base * f, lr=lr, lengths=lengths)[2][:, 6]
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


def persistent_run(model_dir, out, max_grad_norm, target_kl):
    """Child process of the persistent-kernel test: learn at configs[2] through the original entry point, the options
    twin with {0, 0} and with NULL options, then with both guards; every state, metrics row and steps_applied to `out`."""
    from pathlib import Path
    data = baseline_config3(T, E)
    s, a, r, v, d, perms = data
    res = {}
    for tag, kw in (("plain", {}), ("zero", dict(max_grad_norm=0.0, target_kl=0.0)),
                    ("null", dict(max_grad_norm=0.0, target_kl=0.0)),
                    ("guarded", dict(max_grad_norm=max_grad_norm, target_kl=target_kl))):
        m = model(Path(model_dir) / tag, lr=LR_KL)
        if tag == "null":
            with_null_options(m)
        res[tag + "_metrics"] = m.learn(s, a, v, r, d, 0.3, num_epochs=E, batch_size=B, perms=perms, return_metrics=True, **kw)
        for k, x in state(m).items():
            res[tag + "_" + k] = x
        if kw:
            res[tag + "_applied"] = m.last_steps_applied.cpu().numpy()
    np.savez(out, **res)


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
