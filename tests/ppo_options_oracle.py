"""Float64 restatement of the bounded PPO update (cpb_ppo_learn_opts): global gradient-norm clipping as
torch.nn.utils.clip_grad_norm_ does it, and Stable-Baselines3's approximate-KL early stopping, around the minibatch loss
and TF-ApplyAdam of oracle/ppo_oracle.py and oracle/vae_oracle.py.  With both guards off it is oracle.ppo_oracle.learn
step for step (tests/test_ppo_learn_options_cpu.py pins that bit for bit)."""
import numpy as np


def approx_kl(ratio):
    """Stable-Baselines3's approximate KL of the old policy from the new one: mean((r - 1) - log r)."""
    ratio = np.asarray(ratio)
    return np.mean((ratio - 1.0) - np.log(ratio))


def clip_grad_norm(grads, max_norm):
    """torch.nn.utils.clip_grad_norm_ over all tensors of ``grads``: n = sqrt(sum g^2); when max_norm > 0 and
    c = max_norm / (n + 1e-6) < 1 every gradient is multiplied by c.  -> (n, clipped grads); ``grads`` is not changed."""
    norm = np.sqrt(sum(np.sum(np.square(g)) for g in grads.values()))
    if max_norm and max_norm > 0:
        c = max_norm / (norm + 1e-6)
        if c < 1.0:
            return norm, {k: g * c for k, g in grads.items()}
    return norm, dict(grads)


def learn(params, adam_state, states, actions, values, rewards, dones, last_value, low, high,
          gamma=0.99, lam=0.95, lr=1e-4, epsilon=0.2, value_scale=1.0, entropy_scale=0.01,
          num_epochs=3, batch_size=32, perms=None, dtype=np.float64, max_grad_norm=0.0, target_kl=0.0,
          segment_lengths=None, bootstrap_values=None):
    """oracle.ppo_oracle.learn with the guards (0 = off): each minibatch's gradient is clipped to the global norm
    max_grad_norm, and from the first minibatch whose approx_kl exceeds 1.5 * target_kl no Adam step is applied.
    ``segment_lengths`` / ``bootstrap_values``: the rows are several rollouts (cpb_ppo_learn_segments_opts).
    ``params`` and ``adam_state`` are updated in place.  -> (records [steps][7]: the five losses, approx_kl, the pre-clip
    norm; NaN rows after the stop, Adam steps applied)."""
    from oracle import ppo_oracle as po
    from oracle.vae_oracle import adam_apply
    if segment_lengths is None:
        returns, adv_n, _ = po.returns_and_normalised_advantages(rewards, values, last_value, dones, gamma, lam)
    else:
        from ppo_cases import segmented_gae
        returns, adv_n, _ = segmented_gae(rewards, values, bootstrap_values, dones, segment_lengths, gamma, lam)
    states = np.asarray(states, dtype); actions = np.asarray(actions, dtype)
    returns32 = returns.astype(np.float32).astype(dtype)        # the float32 feed of the reference
    adv32 = adv_n.astype(np.float32).astype(dtype)
    old = {k: v.copy() for k, v in params.items()}              # update_old_policy()
    n = states.shape[0]
    records, applied, stopped = [], 0, False
    for e in range(num_epochs):
        idx = np.asarray(perms[e])
        for i in range(int(np.ceil(n / batch_size))):
            if stopped:
                records.append((np.nan,) * 7)
                continue
            mb = idx[i * batch_size:(i + 1) * batch_size]
            out = po.loss_and_grads(params, old, states[mb], actions[mb], returns32[mb], adv32[mb], low, high,
                                    epsilon, value_scale, entropy_scale, True, dtype)
            kl = approx_kl(out["ratio"])
            norm, grads = clip_grad_norm(out["grads"], max_grad_norm)
            records.append((out["policy_loss"], out["value_loss"], out["entropy_loss"], out["loss"], out["mean_ratio"],
                            kl, norm))
            if target_kl and kl > 1.5 * target_kl:
                stopped = True
                continue
            adam_apply(params, grads, adam_state, lr)
            applied += 1
    return np.asarray(records, np.float64).reshape(-1, 7), applied
