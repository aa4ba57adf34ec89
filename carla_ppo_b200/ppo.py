"""Drop-in for the reference's ``ppo.py``: the ``PPO`` class with the same constructor, methods and
attributes, backed by libcarla_ppo_b200.so instead of a TensorFlow session.

Reference surface mirrored (paths relative to the reference repo root):
  * ``PPO.__init__`` hyper-parameters, dirs                   ppo.py:73-190
  * ``init_session / save / load_latest_checkpoint``          ppo.py:192-216
  * ``train`` (ONE minibatch Adam step)                       ppo.py:218-229
  * ``predict`` (greedy / sampled+clipped action, value)      ppo.py:231-251
  * counters, summaries, ``update_old_policy``                ppo.py:253-276

Additive entry point: ``learn(...)`` = the driver's whole update block (train.py:171-207: GAE, returns,
advantage normalisation, theta_old <- theta, epochs x shuffled minibatches) in one C call with no host
round trips.

Additive options of ``learn`` and ``train`` (off by default, which is the reference's update): ``max_grad_norm`` clips the
global L2 norm of each minibatch gradient and ``target_kl`` stops the update once the approximate KL between the new and
the old policy exceeds 1.5 x target_kl (include/carla_ppo_b200.h, "Bounded PPO updates").

Additive constructor arguments ``policy_hidden_sizes`` / ``value_hidden_sizes`` (default: the reference's 500, 300 for
both) size the two trunks independently, 1 to 8 dense + ReLU layers each, like Stable-Baselines3's
``net_arch=dict(pi=[...], vf=[...])``.  Every call goes through the cpb_ppo_spec_* entry points; checkpoints carry the
architecture in their variable names and shapes (``checkpoint_architecture``).

Discrete action spaces (an addition: the reference's policy is always the tanh-squashed Gaussian over a Box):
``action_space`` may be a Discrete(n) (anything with ``.n``) or a MultiDiscrete(nvec) (anything with ``.nvec``): 1 to 4
components of 2 to 64 categories, 64 in all.  The policy head is then a categorical distribution per component
(cpb_ppo_cat_* entry points, include/carla_ppo_b200.h "Categorical policies"); actions are int64 indices, ``predict``
samples with [B, K] uniforms, and checkpoints record the categories (``checkpoint_action_categories``).

Running normalisation (an addition, Stable-Baselines3's VecNormalize): ``normalize_observations`` /
``normalize_rewards`` (with ``clip_obs``, ``clip_reward`` and ``reward_gamma``) give the agent a ``vec_normalize``
(vec_normalize.py) that the actors use to normalise the states and rewards the agent sees.  The checkpoint carries its
statistics (``vec_normalize/*``), and one whose settings differ from the agent's is refused.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Dict, Optional

import numpy as np

from . import _lib
from ._lib import CpbError, PpoCatSpec, PpoConfig, PpoSpec
from .vec_normalize import VecNormalize, blob_normalization

ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8
_METRIC_NAMES = ("train_loss/policy", "train_loss/value", "train_loss/entropy", "train_loss/loss", "train/prob_ratio")
_GUARD_METRIC_NAMES = ("train/approx_kl", "train/grad_norm")     # metric columns 5 and 6 of a guarded update


def learn_options(max_grad_norm=None, target_kl=None):
    """cpb_ppo_learn_options of the two guards (None = off, like 0), or None when both are None."""
    if max_grad_norm is None and target_kl is None:
        return None
    return _lib.PpoLearnOptions(float(max_grad_norm or 0.0), float(target_kl or 0.0))


ARCH_KEYS = ("ppo_architecture/policy_hidden_sizes", "ppo_architecture/value_hidden_sizes")
CATEGORIES_KEY = "ppo_architecture/action_categories"


def action_categories(action_space):
    """The categories (n_1 .. n_K) of a discrete action space -- ``.nvec`` (MultiDiscrete) or ``.n`` (Discrete) -- or None
    for a Box (``.shape`` / ``.low`` / ``.high``).  Raises ValueError outside 1..4 components of 2..64 categories, 64 in
    all."""
    if hasattr(action_space, "nvec"):
        cats = tuple(int(v) for v in np.asarray(action_space.nvec).reshape(-1))
    elif hasattr(action_space, "n"):
        cats = (int(action_space.n),)
    else:
        return None
    if not 1 <= len(cats) <= 4 or min(cats) < 2 or max(cats) > _lib.PPO_MAX_LOGITS or sum(cats) > _lib.PPO_MAX_LOGITS:
        raise ValueError("discrete action spaces take 1 to 4 components of 2 to %d categories, %d in all; got %r"
                         % (_lib.PPO_MAX_LOGITS, _lib.PPO_MAX_LOGITS, cats))
    return cats


def blob_action_categories(blob, scope="policy/"):
    """The categories a checkpoint blob records, or () for a Gaussian one (no record: the reference's).  Raises ValueError
    when the record and the action_logits kernel disagree."""
    if CATEGORIES_KEY not in blob:
        if scope + "action_logits/kernel" in blob:
            raise ValueError("the checkpoint has a categorical head but does not record its categories")
        return ()
    cats = tuple(int(v) for v in np.asarray(blob[CATEGORIES_KEY]).reshape(-1))
    if scope + "action_logits/kernel" not in blob or np.shape(blob[scope + "action_logits/kernel"])[1] != sum(cats):
        raise ValueError("the checkpoint records categories %r, which its action_logits kernel does not have" % (cats,))
    return cats


def _fmt(arch):
    return "policy %s / value %s" % (list(arch[0]), list(arch[1]))


def _inferred_architectures(blob, scope):
    """Every (policy_sizes, value_sizes) that the dense kernels of a blob can be read as, from their names (dense,
    dense_1, ... in creation order: the policy trunk, then the value trunk) and shapes."""
    kernels = []
    while True:
        name = "%sdense%s/kernel" % (scope, "_%d" % len(kernels) if kernels else "")
        if name not in blob:
            break
        kernels.append(np.shape(blob[name]))
    head = scope + ("action_mean/kernel" if scope + "action_mean/kernel" in blob else "action_logits/kernel")
    if len(kernels) < 2 or head not in blob or scope + "value/kernel" not in blob:
        raise ValueError("not a PPO checkpoint: expected %sdense .. dense_N, action_mean (or action_logits) and value kernels"
                         % scope)
    state_dim = kernels[0][0]
    p_last, v_last = np.shape(blob[head])[0], np.shape(blob[scope + "value/kernel"])[0]
    chain = lambda ks: all(ks[i][0] == ks[i - 1][1] for i in range(1, len(ks)))
    out = []
    for n_pol in range(1, len(kernels)):
        pol, val = kernels[:n_pol], kernels[n_pol:]
        if chain(pol) and chain(val) and val[0][0] == state_dim and pol[-1][1] == p_last and val[-1][1] == v_last:
            out.append((tuple(int(k[1]) for k in pol), tuple(int(k[1]) for k in val)))
    if not out:
        raise ValueError("the dense kernels of this checkpoint form no policy / value pair of trunks: %r" % (kernels,))
    return out


def blob_architecture(blob, scope="policy/"):
    """(policy_sizes, value_sizes) of a checkpoint blob.  ``save`` records it (ARCH_KEYS), and the recorded lists must
    agree with the variables' names and shapes.  A checkpoint without the record (the reference's) is read from the names
    and shapes alone; when those fit more than one split between the trunks (a hidden width equal to the state size can
    make the boundary invisible), it is refused rather than guessed.  Raises ValueError."""
    found = _inferred_architectures(blob, scope)
    if ARCH_KEYS[0] in blob and ARCH_KEYS[1] in blob:
        rec = tuple(tuple(int(v) for v in np.asarray(blob[k]).reshape(-1)) for k in ARCH_KEYS)
        if rec not in found:
            raise ValueError("the checkpoint records %s, which its variables do not have (they fit %s)"
                             % (_fmt(rec), " or ".join(_fmt(a) for a in found)))
        return rec
    if len(found) > 1:
        raise ValueError("the checkpoint's variables fit several architectures (%s) and it does not record which one it is"
                         % ", ".join(_fmt(a) for a in found))
    return found[0]


def _latest_checkpoint_prefix(checkpoint_dir):
    """The path prefix that checkpoint_dir's ``checkpoint`` state file names, or None."""
    state = os.path.join(checkpoint_dir, "checkpoint")
    if not os.path.isfile(state):
        return None
    with open(state) as f:
        m = re.search(r'^model_checkpoint_path:\s*"(.*)"', f.read(), re.M)
    if not m:
        return None
    prefix = m.group(1)
    return prefix if os.path.isabs(prefix) else os.path.join(checkpoint_dir, prefix)


def _read_blob(prefix):
    """The variables of the .npz or TF-bundle checkpoint at prefix, or None when neither file exists."""
    if os.path.isfile(prefix + ".npz"):
        return dict(np.load(prefix + ".npz"))
    if os.path.isfile(prefix + ".index"):
        from .tf_bundle import BundleReader
        return BundleReader(prefix).all()
    return None


def checkpoint_architecture(checkpoint_dir):
    """(policy_hidden_sizes, value_hidden_sizes) of the latest checkpoint in checkpoint_dir (a PPO's
    ``checkpoint_dir``), or None when there is none.  Raises ValueError for a file that is not a PPO checkpoint or whose
    architecture is ambiguous (blob_architecture)."""
    prefix = _latest_checkpoint_prefix(checkpoint_dir)
    blob = _read_blob(prefix) if prefix is not None else None
    return None if blob is None else blob_architecture(blob)


def checkpoint_normalization(checkpoint_dir):
    """(normalize_observations, normalize_rewards, clip_obs, clip_reward) of the latest checkpoint in checkpoint_dir,
    (False, False, None, None) for one without normalisation, None when there is no checkpoint."""
    prefix = _latest_checkpoint_prefix(checkpoint_dir)
    blob = _read_blob(prefix) if prefix is not None else None
    if blob is None:
        return None
    return blob_normalization(blob) or (False, False, None, None)


def checkpoint_action_categories(checkpoint_dir):
    """The action categories of the latest checkpoint in checkpoint_dir: a tuple for a categorical agent, () for a
    Gaussian one, None when there is no checkpoint.  Raises ValueError like blob_action_categories."""
    prefix = _latest_checkpoint_prefix(checkpoint_dir)
    blob = _read_blob(prefix) if prefix is not None else None
    return None if blob is None else blob_action_categories(blob)


class PPO:
    def __init__(self, input_shape, action_space, learning_rate=3e-4, lr_decay=0.998, epsilon=0.2,
                 value_scale=0.5, entropy_scale=0.01, initial_std=0.4, model_dir="./", seed=None, device=None,
                 policy_hidden_sizes=_lib.PPO_DEFAULT_HIDDEN, value_hidden_sizes=_lib.PPO_DEFAULT_HIDDEN,
                 normalize_observations=False, normalize_rewards=False, clip_obs=10.0, clip_reward=10.0, reward_gamma=0.99):
        self.policy_hidden_sizes = tuple(int(v) for v in policy_hidden_sizes)
        self.value_hidden_sizes = tuple(int(v) for v in value_hidden_sizes)
        for name, sizes in (("policy_hidden_sizes", self.policy_hidden_sizes), ("value_hidden_sizes", self.value_hidden_sizes)):
            if not 1 <= len(sizes) <= _lib.PPO_MAX_LAYERS or min(sizes) < 1:
                raise ValueError("%s: 1 to %d widths, each >= 1, got %r" % (name, _lib.PPO_MAX_LAYERS, sizes))
        input_shape = tuple(int(v) for v in np.atleast_1d(input_shape))
        if len(input_shape) != 1:
            raise ValueError("PPO expects a flat state vector (reference train.py:85 builds [z_dim + measurements])")
        self.input_shape = input_shape
        self.state_dim = input_shape[0]
        # the running normalisation of the states and rewards the agent sees (None: off, the reference's)
        self.vec_normalize = (VecNormalize(self.state_dim, normalize_observations, normalize_rewards, clip_obs, clip_reward,
                                           reward_gamma) if normalize_observations or normalize_rewards else None)
        self.action_categories = action_categories(action_space)     # None: the reference's Gaussian over a Box
        if self.action_categories is not None:
            self.num_actions = len(self.action_categories)
            self.action_low = self.action_high = np.zeros(self.num_actions, np.float32)
        else:
            self.num_actions = int(action_space.shape[0])
            if self.num_actions > 4:
                raise ValueError("at most 4 action dimensions are supported")
            self.action_low = np.broadcast_to(np.asarray(action_space.low, np.float32), (self.num_actions,)).copy()
            self.action_high = np.broadcast_to(np.asarray(action_space.high, np.float32), (self.num_actions,)).copy()
        self.base_learning_rate = float(learning_rate)
        self.lr_decay = float(lr_decay)
        self.epsilon = float(epsilon)
        self.value_scale = float(value_scale)
        self.entropy_scale = float(entropy_scale)
        self.initial_std = float(initial_std)
        self._seed = seed
        self._device = device

        self.model_dir = model_dir
        self.checkpoint_dir = "{}/checkpoints/".format(self.model_dir)
        self.log_dir = "{}/logs/".format(self.model_dir)
        self.video_dir = "{}/videos/".format(self.model_dir)
        self.dirs = [self.checkpoint_dir, self.log_dir, self.video_dir]
        for d in self.dirs:
            os.makedirs(d, exist_ok=True)

        self.train_step_counter = 0
        self.predict_step_counter = 0
        self.episode_counter = 0
        self.sess = None
        self.train_writer = None
        self._ws = None
        self._pending_metrics = []
        self._pending_applied = []
        self.last_steps_applied = None       # device int32[1]: Adam steps applied by the last guarded learn / train call

    # ------------------------------------------------------------------ session / state
    @property
    def architecture(self):
        """(policy_hidden_sizes, value_hidden_sizes)"""
        return self.policy_hidden_sizes, self.value_hidden_sizes

    def _legacy_widths(self):
        """(hidden1, hidden2) of the cpb_ppo_config that describes this network: its two widths when both trunks are
        the same two layers, else (0, 0) (only a cpb_ppo_spec describes it)."""
        two = len(self.policy_hidden_sizes) == 2 and self.policy_hidden_sizes == self.value_hidden_sizes
        return self.policy_hidden_sizes if two else (0, 0)

    def _cfg(self):
        """The cpb_ppo_config of this agent (hidden1 / hidden2 from _legacy_widths)."""
        cfg = PpoConfig()
        h1, h2 = self._legacy_widths()
        cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = self.state_dim, self.num_actions, h1, h2
        for k in range(4):
            cfg.action_low[k] = float(self.action_low[k]) if k < self.num_actions else 0.0
            cfg.action_high[k] = float(self.action_high[k]) if k < self.num_actions else 0.0
        cfg.epsilon, cfg.value_scale, cfg.entropy_scale = self.epsilon, self.value_scale, self.entropy_scale
        return cfg

    def init_session(self, sess=None, init_logging=True):
        torch = _lib.require_cuda()
        lib = _lib.load()
        self._torch, self._libh = torch, lib
        if self._device is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._device = torch.device(self._device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        dev = self._device
        self._c = self._cfg()
        if (self._c.hidden1, self._c.hidden2) != tuple(self._legacy_widths()):
            # a subclass that sizes the network through _cfg(), as the two-width interface did: its widths, both trunks
            self.policy_hidden_sizes = self.value_hidden_sizes = (int(self._c.hidden1), int(self._c.hidden2))
        if self.action_categories is None:
            self._spec = PpoSpec.of(self._c, self.policy_hidden_sizes, self.value_hidden_sizes)
            self._api = "cpb_ppo_spec_"
        else:
            self._spec = PpoCatSpec.of(self._c, self.policy_hidden_sizes, self.value_hidden_sizes, self.action_categories)
            self._api = "cpb_ppo_cat_"
        api = lambda name: getattr(lib, self._api + name)
        n = _lib.check(api("num_tensors")(C.byref(self._spec)), self._api + "num_tensors")
        offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (2 * n))()
        total = C.c_int64()
        _lib.check(api("layout")(C.byref(self._spec), offs, sizes, shapes, C.byref(total)), self._api + "layout")
        self._names = [api("tensor_name")(C.byref(self._spec), i).decode() for i in range(n)]
        self._offsets = {self._names[i]: int(offs[i]) for i in range(n)}
        self._shapes = {self._names[i]: tuple(int(s) for s in shapes[2 * i:2 * i + 2] if s > 0) for i in range(n)}
        self._total = int(total.value)
        z = lambda: torch.zeros(self._total, dtype=torch.float32, device=dev)
        self.params, self.params_old, self.grads, self.adam_m, self.adam_v = z(), z(), z(), z(), z()
        self.adam_powers = torch.tensor([ADAM_BETA1, ADAM_BETA2], dtype=torch.float32, device=dev)
        self._lr_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self._rng = np.random.RandomState(self._seed)
        w = self._initial_weights()
        self.set_weights(w, w)
        self._sync_lr()
        if self.vec_normalize is not None:
            self.vec_normalize.init_session(torch, lib, dev, self._stream)
        self.sess = self
        if init_logging:
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.train_writer = SummaryWriter(self.log_dir)
            except Exception as e:
                print("carla_ppo_b200: TensorBoard logging disabled (%s)" % e)

    def _initial_weights(self) -> Dict[str, np.ndarray]:
        """tf.layers.dense defaults (glorot uniform / zeros); action_mean kernel = variance_scaling(0.1)
        truncated normal (ppo.py:44-47); action_logstd = log(initial_std) (ppo.py:49).  A categorical head's
        action_logits kernel is drawn like action_mean's (a near-uniform initial policy)."""
        rng = np.random.RandomState(self._seed if self._seed is not None else np.random.randint(0, 2 ** 31 - 1))
        out = {}
        for name in self._names:
            shape = self._shapes[name]
            if name == "action_logstd":
                out[name] = np.full(shape, np.log(self.initial_std), np.float32)
            elif name.endswith("bias"):
                out[name] = np.zeros(shape, np.float32)
            elif name in ("action_mean/kernel", "action_logits/kernel"):
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

    def _flatten(self, weights) -> np.ndarray:
        host = np.zeros(self._total, np.float32)
        for name in self._names:
            w = np.asarray(weights[name], np.float32).reshape(self._shapes[name])
            o = self._offsets[name]
            host[o:o + w.size] = w.ravel()
        return host

    def _unflatten(self, flat) -> Dict[str, np.ndarray]:
        host = flat.detach().cpu().numpy()
        return {n: host[self._offsets[n]:self._offsets[n] + int(np.prod(self._shapes[n]))].reshape(self._shapes[n]).copy()
                for n in self._names}

    def set_weights(self, policy, policy_old=None, adam_m=None, adam_v=None, powers=None):
        torch = self._torch
        self.params.copy_(torch.from_numpy(self._flatten(policy)))
        if policy_old is not None:
            self.params_old.copy_(torch.from_numpy(self._flatten(policy_old)))
        if adam_m is not None:
            self.adam_m.copy_(torch.from_numpy(self._flatten(adam_m)))
        if adam_v is not None:
            self.adam_v.copy_(torch.from_numpy(self._flatten(adam_v)))
        if powers is not None:
            self.adam_powers.copy_(torch.tensor([float(powers[0]), float(powers[1])], dtype=torch.float32))

    def get_weights(self):
        return self._unflatten(self.params)

    def get_old_weights(self):
        return self._unflatten(self.params_old)

    def get_grads(self):
        return self._unflatten(self.grads)

    @property
    def learning_rate(self):
        """exponential_decay(learning_rate, episode_counter, 1, lr_decay, staircase) (ppo.py:142)."""
        return np.float32(self.base_learning_rate) * np.float32(self.lr_decay) ** np.float32(self.episode_counter)

    def _sync_lr(self):
        self._lr_dev.fill_(float(self.learning_rate))

    def _require_session(self):
        if self.sess is None:
            raise CpbError("init_session() has not been called")

    def _stream(self):
        return _lib.current_stream_handle(self._device)

    def _call(self, name, *args):
        """C entry point with this model's device current (the library launches on the CURRENT CUDA device)."""
        with self._torch.cuda.device(self._device):
            return _lib.check(getattr(self._libh, name)(*args), name)

    def _workspace(self, max_batch, horizon=0):
        need = getattr(self._libh, self._api + "workspace_bytes")(C.byref(self._spec), int(max_batch), int(horizon))
        _lib.check(need, self._api + "workspace_bytes")
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = self._torch.empty(int(need), dtype=self._torch.uint8, device=self._device)
        return self._ws

    def _actions(self, a, rows=-1):
        """Taken actions as a device float32 [rows, K] tensor.  A categorical agent takes integer indices; host arrays are
        checked (ValueError for a non-integer or out-of-range index), device tensors are passed as they are (the kernels
        clamp every index into its component's range)."""
        torch = self._torch
        if self.action_categories is not None and not isinstance(a, torch.Tensor):
            host = np.asarray(a, np.float64).reshape(rows, self.num_actions)
            if not np.all(np.isfinite(host)) or np.any(host != np.round(host)):
                raise ValueError("discrete actions must be integer indices")
            if np.any(host < 0) or np.any(host >= np.asarray(self.action_categories)):
                raise ValueError("discrete actions must lie in [0, n_k) for categories %r" % (self.action_categories,))
        return self._dev(a, torch.float32).reshape(rows, self.num_actions)

    def _dev(self, a, dtype):
        torch = self._torch
        if isinstance(a, torch.Tensor):
            return a.to(self._device, dtype).contiguous()
        np_dtype = {torch.float32: np.float32, torch.float64: np.float64, torch.int32: np.int32}[dtype]
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np_dtype))).to(self._device)

    # ------------------------------------------------------------------ checkpoints
    def save(self, tf_format=False):
        """.npz checkpoint + ``checkpoint`` state file (ppo.py:202-205); ``tf_format=True`` writes a TF-V2 tensor bundle
        with the reference's variable names instead (readable by the reference's ``saver.restore``)."""
        self._require_session()
        step = int(self.episode_counter)
        prefix = os.path.join(self.checkpoint_dir, "model.ckpt-%d" % step)
        blob = {}
        for k, v in self.get_weights().items():
            blob["policy/" + k] = v
        for k, v in self.get_old_weights().items():
            blob["policy_old/" + k] = v
        for k, v in self._unflatten(self.adam_m).items():
            blob["policy/%s/Adam" % k] = v
        for k, v in self._unflatten(self.adam_v).items():
            blob["policy/%s/Adam_1" % k] = v
        pw = self.adam_powers.cpu().numpy()
        blob["beta1_power"], blob["beta2_power"] = pw[0], pw[1]
        blob["episode_counter"] = np.int32(self.episode_counter)
        blob["train_step_counter"] = np.int32(self.train_step_counter)
        blob["predict_step_counter"] = np.int32(self.predict_step_counter)
        for key, sizes in zip(ARCH_KEYS, self.architecture):
            blob[key] = np.asarray(sizes, np.int32)
        if self.action_categories is not None:
            blob[CATEGORIES_KEY] = np.asarray(self.action_categories, np.int32)
        if self.vec_normalize is not None:
            blob.update(self.vec_normalize.state_dict())
        if tf_format:
            from .tf_bundle import write_bundle
            write_bundle(prefix, {k: np.asarray(v) for k, v in blob.items()})
        else:
            np.savez(prefix + ".npz", **blob)
        state = os.path.join(self.checkpoint_dir, "checkpoint")
        kept = []
        if os.path.isfile(state):
            with open(state) as f:
                kept = re.findall(r'^all_model_checkpoint_paths:\s*"(.*)"', f.read(), re.M)
        name = os.path.basename(prefix)
        kept = [k for k in kept if k != name] + [name]
        for old in kept[:-5]:
            for ext in (".npz", ".index", ".data-00000-of-00001"):
                try:
                    os.remove(os.path.join(self.checkpoint_dir, old + ext))
                except OSError:
                    pass
        with open(state, "w") as f:
            f.write('model_checkpoint_path: "%s"\n' % name)
            for k in kept[-5:]:
                f.write('all_model_checkpoint_paths: "%s"\n' % k)
        print("Model checkpoint saved to {}".format(prefix))

    def load_latest_checkpoint(self):
        """True / False (restore raised) / None (no checkpoint), like ppo.py:207-216."""
        self._require_session()
        prefix = _latest_checkpoint_prefix(self.checkpoint_dir)
        if prefix is None:
            return None
        try:
            blob = _read_blob(prefix)
            if blob is None:
                return None
            self.load_blob(blob)
            print("Model checkpoint restored from {}".format(prefix))
            return True
        except Exception as e:
            print(e)
            return False

    def load_blob(self, blob):
        """Restore from a checkpoint's variables; a checkpoint of another architecture, action space or normalisation
        setting is refused (ValueError)."""
        found = blob_architecture(blob)
        if found != self.architecture:
            raise ValueError("checkpoint architecture %s does not match this PPO's %s" % (_fmt(found), _fmt(self.architecture)))
        cats = blob_action_categories(blob)
        if cats != (self.action_categories or ()):
            kind = lambda c: "categories %r" % (c,) if c else "a Gaussian policy"
            raise ValueError("the checkpoint has %s, this PPO %s" % (kind(cats), kind(self.action_categories)))
        found_norm = blob_normalization(blob)
        mine = None if self.vec_normalize is None else self.vec_normalize.settings
        if found_norm != mine:
            kind = lambda n: ("no normalisation" if n is None else "normalize_observations=%s, normalize_rewards=%s, "
                              "clip_obs=%g, clip_reward=%g" % n)
            raise ValueError("the checkpoint has %s, this PPO %s" % (kind(found_norm), kind(mine)))
        pol = {n: blob["policy/" + n] for n in self._names}
        old = {n: blob["policy_old/" + n] for n in self._names}
        m_ = v_ = pw = None
        if ("policy/%s/Adam" % self._names[0]) in blob:
            m_ = {n: blob["policy/%s/Adam" % n] for n in self._names}
            v_ = {n: blob["policy/%s/Adam_1" % n] for n in self._names}
            pw = (float(blob["beta1_power"]), float(blob["beta2_power"]))
        self.set_weights(pol, old, m_, v_, pw)
        if self.vec_normalize is not None:
            self.vec_normalize.load_state_dict(blob)
        for attr in ("episode_counter", "train_step_counter", "predict_step_counter"):
            if attr in blob:
                setattr(self, attr, int(blob[attr]))
        self._sync_lr()

    # ------------------------------------------------------------------ hot path
    def train(self, input_states, taken_actions, returns, advantage, max_grad_norm=None, target_kl=None, stop=None):
        """ONE minibatch Adam step (ppo.py:218-229).  Metrics stay on the device until the next
        write_episodic_summaries().

        ``max_grad_norm`` / ``target_kl`` (None = off): the guards of learn() on this step; ``stop`` (a device int32[1]
        from new_stop_word(), zeroed once per update) carries the KL stop from step to step, so that a loop of train calls
        stops exactly as learn() does, without a host sync.  With any of the three, the metrics are 7 wide and the step
        goes through cpb_ppo_train_step_opts."""
        self._require_session()
        torch = self._torch
        s = self._dev(input_states, torch.float32).reshape(-1, self.state_dim)
        a = self._actions(taken_actions)
        r = self._dev(returns, torch.float32).reshape(-1)
        adv = self._dev(advantage, torch.float32).reshape(-1)
        b = s.shape[0]
        if not (a.shape[0] == r.shape[0] == adv.shape[0] == b):
            raise ValueError("train(): inconsistent batch sizes")
        opts = learn_options(max_grad_norm, target_kl)
        if opts is None and stop is not None:
            opts = learn_options(0.0, 0.0)
        metrics = torch.empty(5 if opts is None else 7, dtype=torch.float32, device=self._device)
        ws = self._workspace(b)
        if opts is None:
            self._call(self._api + "train_step",
                C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(self.grads),
                _lib.ptr(self.adam_m), _lib.ptr(self.adam_v), _lib.ptr(self.adam_powers), _lib.ptr(self._lr_dev),
                _lib.ptr(s), _lib.ptr(a), _lib.ptr(r), _lib.ptr(adv), None, b, _lib.ptr(metrics), _lib.ptr(ws),
                ws.numel(), self._stream())
        else:
            applied = torch.empty(1, dtype=torch.int32, device=self._device)
            self._call(self._api + "train_step_opts",
                C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(self.grads),
                _lib.ptr(self.adam_m), _lib.ptr(self.adam_v), _lib.ptr(self.adam_powers), _lib.ptr(self._lr_dev),
                _lib.ptr(s), _lib.ptr(a), _lib.ptr(r), _lib.ptr(adv), None, b, _lib.ptr(metrics), C.byref(opts),
                _lib.ptr(stop), _lib.ptr(applied), _lib.ptr(ws), ws.numel(), self._stream())
            self._pending_applied.append(applied)
            self.last_steps_applied = applied
        self._pending_metrics.append(metrics)
        self.train_step_counter += 1
        return metrics

    def new_stop_word(self):
        """A zeroed device stop word for one update of train(..., stop=...) steps."""
        self._require_session()
        return self._torch.zeros(1, dtype=self._torch.int32, device=self._device)

    def loss_and_grads(self, input_states, taken_actions, returns, advantage):
        """Loss + gradients only (no Adam): returns (metrics[5] ndarray, {name: grad})."""
        self._require_session()
        torch = self._torch
        s = self._dev(input_states, torch.float32).reshape(-1, self.state_dim)
        a = self._actions(taken_actions)
        r = self._dev(returns, torch.float32).reshape(-1)
        adv = self._dev(advantage, torch.float32).reshape(-1)
        b = s.shape[0]
        metrics = torch.empty(5, dtype=torch.float32, device=self._device)
        ws = self._workspace(b)
        self._call(self._api + "loss_grad",
            C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(s), _lib.ptr(a), _lib.ptr(r),
            _lib.ptr(adv), None, b, _lib.ptr(self.grads), _lib.ptr(metrics), _lib.ptr(ws), ws.numel(),
            self._stream())
        return metrics.cpu().numpy(), self.get_grads()

    def predict(self, input_states, greedy=False, write_to_summary=False, noise=None):
        """-> (action, value); squeezed when a single state is given (ppo.py:231-251).  ``noise`` (optional
        [B,A] standard-normal draws) makes the sampled action reproducible.  A categorical agent returns int64 indices
        [B,K]: the most likely category of each component when greedy, else the inverse-CDF draw of ``noise`` ([B,K]
        uniforms in [0, 1), default self._rng.rand)."""
        self._require_session()
        torch = self._torch
        x = np.asarray(input_states, dtype=np.float32)
        if x.ndim != 2:
            x = x[None]
        b, a_dim = x.shape[0], self.num_actions
        if greedy:
            packed = x
        else:
            draw = self._rng.randn if self.action_categories is None else self._rng.rand
            eps = draw(b, a_dim).astype(np.float32) if noise is None else np.asarray(noise, np.float32).reshape(b, a_dim)
            packed = np.concatenate([x.reshape(-1), eps.reshape(-1)])
        dev = torch.from_numpy(np.ascontiguousarray(packed).reshape(-1)).to(self._device)
        s = dev[:b * self.state_dim]
        nz = None if greedy else dev[b * self.state_dim:]
        out = torch.empty(b * (a_dim + 1), dtype=torch.float32, device=self._device)
        ws = self._workspace(b)
        self._call(self._api + "forward", C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(s), b, _lib.ptr(nz),
                                              _lib.ptr(out), _lib.ptr(out[b * a_dim:]), _lib.ptr(ws), ws.numel(),
                                              self._stream())
        host = out.cpu().numpy()
        action, value = host[:b * a_dim].reshape(b, a_dim), host[b * a_dim:]
        if self.action_categories is not None:
            action = action.astype(np.int64)
        if write_to_summary:
            if self.train_writer is not None:
                for i in range(a_dim):
                    self.train_writer.add_scalar("predict_actor/action_%d/sampled_action" % i, float(action[0, i]),
                                                 self.predict_step_counter)
            self.predict_step_counter += 1
        if b == 1:
            return action[0], value[0]
        return action, value

    def update_old_policy(self):
        """theta_old <- theta (ppo.py:147, 275-276)."""
        self._require_session()
        self.params_old.copy_(self.params)

    def learn(self, states, actions, values, rewards, dones, last_value, gamma=0.99, lam=0.95, num_epochs=3,
              batch_size=32, perms=None, return_metrics=False, segment_lengths=None, max_grad_norm=None, target_kl=None):
        """train.py:171-207 in one C call: compute_gae -> returns -> normalised advantages ->
        update_old_policy -> num_epochs x ceil(T/batch_size) minibatch steps.  ``perms`` ([num_epochs, T]
        index orders) defaults to np.random permutations like the reference's np.random.shuffle.

        ``segment_lengths`` (S lengths, each >= 1, summing to T): the rows are S environments' rollouts concatenated in
        that order and ``last_value`` holds their S bootstrap values.  GAE runs per segment, the advantages are
        normalised once over all T rows, and the minibatches draw from all of them (cpb_ppo_learn_segments).

        ``max_grad_norm`` (clip the global L2 norm of each minibatch gradient) and ``target_kl`` (skip every Adam step from
        the first minibatch whose approximate KL exceeds 1.5 x target_kl): None = off.  With either, the update runs
        through the *_opts entry points, metrics rows are 7 wide (+ approx_kl, pre-clip grad_norm; NaN after a stop) and
        ``last_steps_applied`` holds the number of Adam steps applied."""
        if segment_lengths is not None:
            rows = int(np.prod(states.shape if hasattr(states, "shape") else np.shape(states))) // self.state_dim
            lengths = [int(n) for n in segment_lengths]
            if not lengths or min(lengths) < 1 or sum(lengths) != rows:
                raise ValueError("learn(): segment_lengths must be >= 1 each and sum to the %d rows, got %r" % (rows, lengths))
            boot = np.asarray(last_value, np.float64).reshape(-1)
            if boot.shape[0] != len(lengths):
                raise ValueError("learn(): %d segments need as many bootstrap values, got %d" % (len(lengths), boot.shape[0]))
        self._require_session()
        torch = self._torch
        s = self._dev(states, torch.float32).reshape(-1, self.state_dim)
        t_len = s.shape[0]
        a = self._actions(actions, t_len)
        r = self._dev(rewards, torch.float64).reshape(t_len)
        v = self._dev(values, torch.float64).reshape(t_len)
        d = self._dev(np.asarray(dones, dtype=np.float64) if not isinstance(dones, torch.Tensor) else dones, torch.float64).reshape(t_len)
        if perms is None:
            perms = np.stack([np.random.permutation(t_len) for _ in range(num_epochs)]) if num_epochs else np.zeros((0, t_len))
        if num_epochs == 0:
            p = None                       # nothing to index: the C entry accepts perms == NULL for zero epochs
        elif isinstance(perms, torch.Tensor):
            p = perms.to(self._device, torch.int32).reshape(num_epochs, t_len).contiguous()
        else:
            p = self._dev(np.asarray(perms).reshape(num_epochs, t_len), torch.int32)
        nmb = -(-t_len // batch_size)
        opts = learn_options(max_grad_norm, target_kl)
        ncol = 5 if opts is None else 7
        metrics = torch.empty(max(num_epochs * nmb, 1), ncol, dtype=torch.float32, device=self._device)
        ws = self._workspace(min(batch_size, t_len), t_len)
        if opts is not None:
            applied = torch.empty(1, dtype=torch.int32, device=self._device)
            common = (C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(self.grads),
                      _lib.ptr(self.adam_m), _lib.ptr(self.adam_v), _lib.ptr(self.adam_powers), _lib.ptr(self._lr_dev),
                      _lib.ptr(s), _lib.ptr(a), _lib.ptr(r), _lib.ptr(v))
            tail = (float(gamma), float(lam), int(num_epochs), int(batch_size), _lib.ptr(p), _lib.ptr(metrics),
                    C.byref(opts), _lib.ptr(applied), _lib.ptr(ws), ws.numel(), self._stream())
            if segment_lengths is None:
                self._call(self._api + "learn_opts", *common, float(last_value), _lib.ptr(d), t_len, *tail)
            else:
                b = self._dev(boot, torch.float64)
                offsets = self._dev(np.concatenate([[0], np.cumsum(lengths)]), torch.int32)
                self._call(self._api + "learn_segments_opts", *common, _lib.ptr(b), _lib.ptr(d), _lib.ptr(offsets),
                           len(lengths), t_len, *tail)
            self._pending_applied.append(applied)
            self.last_steps_applied = applied
        elif segment_lengths is None:
            self._call(self._api + "learn",
                C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(self.grads),
                _lib.ptr(self.adam_m), _lib.ptr(self.adam_v), _lib.ptr(self.adam_powers), _lib.ptr(self._lr_dev),
                _lib.ptr(s), _lib.ptr(a), _lib.ptr(r), _lib.ptr(v), float(last_value), _lib.ptr(d), t_len, float(gamma),
                float(lam), int(num_epochs), int(batch_size), _lib.ptr(p), _lib.ptr(metrics), _lib.ptr(ws), ws.numel(),
                self._stream())
        else:
            b = self._dev(boot, torch.float64)
            offsets = self._dev(np.concatenate([[0], np.cumsum(lengths)]), torch.int32)
            self._call(self._api + "learn_segments",
                C.byref(self._spec), _lib.ptr(self.params), _lib.ptr(self.params_old), _lib.ptr(self.grads),
                _lib.ptr(self.adam_m), _lib.ptr(self.adam_v), _lib.ptr(self.adam_powers), _lib.ptr(self._lr_dev),
                _lib.ptr(s), _lib.ptr(a), _lib.ptr(r), _lib.ptr(v), _lib.ptr(b), _lib.ptr(d), _lib.ptr(offsets),
                len(lengths), t_len, float(gamma), float(lam), int(num_epochs), int(batch_size), _lib.ptr(p),
                _lib.ptr(metrics), _lib.ptr(ws), ws.numel(), self._stream())
        self.train_step_counter += num_epochs * nmb
        self._pending_metrics.append(metrics[:num_epochs * nmb])
        if return_metrics:
            return metrics[:num_epochs * nmb].cpu().numpy().reshape(num_epochs * nmb, ncol)
        return None

    # ------------------------------------------------------------------ counters / summaries
    def get_episode_idx(self):
        return int(self.episode_counter)

    def get_train_step_idx(self):
        return int(self.train_step_counter)

    def get_predict_step_idx(self):
        return int(self.predict_step_counter)

    def write_value_to_summary(self, summary_name, value, step):
        if self.train_writer is not None:
            self.train_writer.add_scalar(summary_name, float(value), int(step))

    def write_dict_to_summary(self, summary_name, params, step):
        if self.train_writer is not None:
            self.train_writer.add_text(summary_name, "\n".join("%s: %s" % (k, v) for k, v in params.items()), int(step))

    def write_episodic_summaries(self):
        """Episodic means of the per-minibatch metrics, then episode_counter += 1 (ppo.py:271-273) -- which is
        what decays the learning rate.  After guarded updates the means cover the evaluated rows only (a KL stop leaves
        NaN rows), and train/approx_kl, train/grad_norm and train/updates_applied (Adam steps applied) are added."""
        if self._pending_metrics:
            torch = self._torch
            guarded = [m.reshape(-1, 7) for m in self._pending_metrics if m.shape[-1] == 7]
            if not guarded:
                allm = torch.cat([m.reshape(-1, 5) for m in self._pending_metrics]).double().mean(dim=0).cpu().numpy()
                extra = []
            else:
                rows = torch.cat([m.reshape(-1, m.shape[-1])[:, :5] for m in self._pending_metrics]).double()
                allm = rows[~torch.isnan(rows[:, 0])].mean(dim=0).cpu().numpy()
                g = torch.cat(guarded).double()
                kl_norm = g[~torch.isnan(g[:, 0])][:, 5:7].mean(dim=0).cpu().numpy()
                unguarded_steps = sum(m.reshape(-1, 5).shape[0] for m in self._pending_metrics if m.shape[-1] == 5)
                applied = int(torch.cat(self._pending_applied).sum().item()) + unguarded_steps
                extra = list(zip(_GUARD_METRIC_NAMES, kl_norm)) + [("train/updates_applied", applied)]
            if self.train_writer is not None:
                for name, val in list(zip(_METRIC_NAMES, allm)) + extra:
                    self.train_writer.add_scalar(name, float(val), self.episode_counter)
                self.train_writer.add_scalar("train/learning_rate", float(self.learning_rate), self.episode_counter)
            self._pending_metrics = []
            self._pending_applied = []
        self.episode_counter += 1
        self._sync_lr()
