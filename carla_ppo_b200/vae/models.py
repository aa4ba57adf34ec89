"""Drop-in for the reference's ``vae/models.py``: same class names, constructor arguments, methods,
attributes and NumPy-in / NumPy-out conventions, backed by libcarla_ppo_b200.so (hand-written sm_90a
CUDA behind a C ABI) instead of a TensorFlow session.

Reference surface mirrored here (paths relative to the reference repo root):
  * loss selectors ``bce_loss`` / ``bce_loss_v2`` / ``mse_loss``      vae/models.py:11-22
  * ``VAE.__init__`` keyword surface, dirs, ``training`` switch      vae/models.py:38-159
  * ``init_session / save / load_latest_checkpoint``                 vae/models.py:161-186
  * ``generate_from_latent / reconstruct / encode / get_step_idx``   vae/models.py:188-205
  * ``train_one_epoch / evaluate``                                   vae/models.py:207-231
  * ``ConvVAE`` (4x conv 4x4 s2 -> heads -> dense -> 4x deconv)      vae/models.py:233-268

Additive entry points (not in the reference): ``decode`` (= generate_from_latent), ``train_step`` /
``eval_step`` (one minibatch on device or host buffers, noise as an input), data-parallel training
over torch.distributed (one NCCL all-reduce of the flat gradient per step).
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import Dict, Optional

import numpy as np

from .. import _lib
from .._lib import CpbError, MlpVaeConfig, MlpVaeSpec, VaeConfig, VaeSpec


# ----------------------------------------------------------------------------- loss selectors
def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * np.asarray(x, dtype=np.float64)))


def bce_loss(labels, logits, targets):
    """tf.nn.sigmoid_cross_entropy_with_logits (vae/models.py:11-15).  Passed as ``loss_fn=``; the CUDA
    path keys on ``.cpb_loss_type``; calling it evaluates the same formula on host arrays."""
    x = np.asarray(logits, np.float64); y = np.asarray(labels, np.float64)
    return np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))


def bce_loss_v2(labels, logits, targets, epsilon=1e-10):
    y = np.asarray(labels, np.float64); t = np.asarray(targets, np.float64)
    return -(y * np.log(epsilon + t) + (1 - y) * np.log(epsilon + 1 - t))


def mse_loss(labels, logits, targets):
    return (np.asarray(labels, np.float64) - np.asarray(targets, np.float64)) ** 2


bce_loss.cpb_loss_type = _lib.LOSS_BCE
bce_loss_v2.cpb_loss_type = _lib.LOSS_BCE_V2
mse_loss.cpb_loss_type = _lib.LOSS_MSE
_LOSS_BY_NAME = {"bce": bce_loss, "bce_v2": bce_loss_v2, "mse": mse_loss}

ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8


def _loss_type(loss_fn) -> int:
    if isinstance(loss_fn, str):
        loss_fn = _LOSS_BY_NAME[loss_fn]
    lt = getattr(loss_fn, "cpb_loss_type", None)
    if lt is None:
        raise ValueError("loss_fn must be one of bce_loss, bce_loss_v2, mse_loss (arbitrary Python losses "
                         "cannot run inside the fused CUDA loss kernel)")
    return lt


# ----------------------------------------------------------------------------- data-parallel host logic
def dp_noise_rows(torch, generator, batch, z_dim, rank, world, device):
    """This rank's rows of the noise the GLOBAL batch draws: all ranks hold the same generator state, draw
    [world*batch, z] and keep rows [rank*batch, (rank+1)*batch) -- together exactly the single-process draw."""
    full = torch.randn(batch * world, z_dim, generator=generator, device=device, dtype=torch.float32)
    return full[rank * batch:(rank + 1) * batch].contiguous()


def dp_shared_permutation(torch, dist, indices, device):
    """Every rank adopts rank 0's epoch permutation (ranks seed np.random independently)."""
    perm = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.int64)).to(device)
    dist.broadcast(perm, 0)
    return perm.cpu().numpy()


FRAME_MIN, FRAME_MAX = 48, 512


def frame_rule_error(height, width):
    """None when the ConvVAE takes frames of height x width, else the refusal text (the library's, cpb_vae_spec_*): the
    reference's decoder maps the encoder output back to exactly H x W only for multiples of 16 (vae/models.py:265)."""
    if all(FRAME_MIN <= v <= FRAME_MAX and v % 16 == 0 for v in (height, width)):
        return None
    return "frame %dx%d: height and width must each be a multiple of 16 in [48, 512]" % (height, width)


def encoded_hw(height, width):
    """The encoder's output [H4, W4] (four 4x4 stride-2 VALID convolutions)."""
    for _ in range(4):
        height, width = (height - 4) // 2 + 1, (width - 4) // 2 + 1
    return height, width


def recorded_source_shape(checkpoint_dir):
    """The source_shape the latest .npz checkpoint under checkpoint_dir recorded (``vae/source_shape``), or None: no
    checkpoint, a TF bundle, or a checkpoint written before the shape was recorded."""
    state = os.path.join(checkpoint_dir, "checkpoint")
    if not os.path.isfile(state):
        return None
    with open(state) as f:
        m = re.search(r'^model_checkpoint_path:\s*"(.*)"', f.read(), re.M)
    if not m:
        return None
    prefix = m.group(1) if os.path.isabs(m.group(1)) else os.path.join(checkpoint_dir, m.group(1))
    if not os.path.isfile(prefix + ".npz"):
        return None
    with np.load(prefix + ".npz") as blob:
        return tuple(int(v) for v in blob["vae/source_shape"]) if "vae/source_shape" in blob else None


class _Placeholder:
    """Stands in for the TF tensors callers only inspect (``vae.sample.shape[1]``, inspect_vae.py:100)."""

    def __init__(self, shape, name):
        self.shape = tuple(shape)
        self.name = name


class VAE:
    """Base class.  Frames are source [H,W,3], target [H,W,Ct]: the ConvVAE takes every H and W that are multiples of 16
    in [48, 512], the MlpVAE the reference's 80x160."""

    # C entry points of the architecture (ConvVAE: cpb_vae_spec_*, MlpVAE: cpb_mlpvae_spec_*; identical argument lists)
    _API = {"num_tensors": "cpb_vae_num_tensors", "tensor_name": "cpb_vae_tensor_name", "encode": "cpb_vae_spec_encode",
            "decode": "cpb_vae_spec_decode", "forward": "cpb_vae_spec_forward", "loss_grad": "cpb_vae_spec_loss_grad",
            "encode_predict": "cpb_vae_spec_encode_predict"}
    _HOST_STEP = True        # cpb_vae_train_step_host exists for this architecture

    def __init__(self, source_shape, target_shape, build_encoder_fn=None, build_decoder_fn=None,
                 z_dim=512, beta=1.0, learning_rate=1e-4, lr_decay=0.98, kl_tolerance=0.0,
                 model_dir=".", loss_fn=bce_loss, training=True, reuse=None, seed=None,
                 data_parallel=False, device=None, resident_dataset=True, **kwargs):
        # unknown kwargs (e.g. models_dir="vae", vae_common.py:21) are swallowed like the reference does
        self.source_shape = tuple(int(v) for v in source_shape)
        self.target_shape = tuple(int(v) for v in (source_shape if target_shape is None else target_shape))
        self._check_shapes()
        self.z_dim = int(z_dim)
        self.beta = float(beta)
        self.kl_tolerance = float(kl_tolerance)
        self.base_learning_rate = float(learning_rate)
        self.lr_decay = float(lr_decay)
        self.training = bool(training)
        self.loss_fn = loss_fn
        self.loss_type = _loss_type(loss_fn)
        self.data_parallel = bool(data_parallel)
        self._resident_dataset = bool(resident_dataset)
        self._seed = seed
        self._device = device

        self.model_dir = model_dir
        self.checkpoint_dir = "{}/checkpoints/".format(self.model_dir)
        self.log_dir = "{}/logs/".format(self.model_dir)
        self.dirs = [self.checkpoint_dir, self.log_dir]
        for d in self.dirs:
            os.makedirs(d, exist_ok=True)

        # attributes callers inspect
        self.source_states = _Placeholder((None,) + self.source_shape, "source_state_placeholder")
        self.target_states = _Placeholder((None,) + self.target_shape, "target_state_placeholder")
        self.sample = _Placeholder((None, self.z_dim), "sample")
        self.encoded_shape = encoded_hw(*self.source_shape[:2]) + (256,)

        self.sess = None
        self.step_idx = 0
        self._ws = {}
        self._dataset_cache = {}
        self.train_writer = self.val_writer = None
        self._last_metrics = (float("nan"), float("nan"))

    # ------------------------------------------------------------------ session / state
    def init_session(self, sess=None, init_logging=True):
        """Allocates device state and initialises it (glorot-uniform kernels, zero biases: the tf.layers
        defaults the reference relies on).  ``sess`` is accepted and ignored."""
        torch = _lib.require_cuda()
        lib = _lib.load()
        self._torch, self._libh = torch, lib
        if self._device is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        self._device = torch.device(self._device)
        if self._device.index is None:
            self._device = torch.device("cuda", torch.cuda.current_device())
        dev = self._device
        self._names = self._tensor_names(lib)
        n = len(self._names)
        offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (4 * n))()
        total = C.c_int64()
        self._query_layout(lib, offs, sizes, shapes, total)
        self._offsets = {self._names[i]: int(offs[i]) for i in range(n)}
        self._shapes = {self._names[i]: tuple(int(s) for s in shapes[4 * i:4 * i + 4] if s > 0) for i in range(n)}
        self._total = int(total.value)

        self.params = torch.zeros(self._total, dtype=torch.float32, device=dev)
        if self.training:
            # gradients + [recon, kl] in ONE buffer so that data-parallel training needs one all-reduce
            self._gradbuf = torch.zeros(self._total + 64, dtype=torch.float32, device=dev)
            self.grads = self._gradbuf[:self._total]
            self._losses = self._gradbuf[self._total:self._total + 2]
            self.adam_m = torch.zeros(self._total, dtype=torch.float32, device=dev)
            self.adam_v = torch.zeros(self._total, dtype=torch.float32, device=dev)
            self.adam_powers = torch.tensor([ADAM_BETA1, ADAM_BETA2], dtype=torch.float32, device=dev)
        else:
            self._losses = torch.zeros(2, dtype=torch.float32, device=dev)
        self._flags = torch.zeros(1, dtype=torch.int32, device=dev)
        self._noise_gen = torch.Generator(device=dev)
        self._noise_gen.manual_seed(0 if self._seed is None else int(self._seed))
        self.set_weights(self._initial_weights())      # (+ broadcast from rank 0 when data_parallel)
        self.sess = self            # truthy stand-in; some callers test `vae.sess`
        self.step_idx = 0
        if init_logging:
            self._init_logging()

    def _check_shapes(self):
        if len(self.source_shape) != 3 or self.source_shape[2] != 3:
            raise ValueError("source_shape must be (height, width, 3), got %r" % (self.source_shape,))
        err = frame_rule_error(*self.source_shape[:2])
        if err is not None:
            raise ValueError(err)
        h, w = self.source_shape[:2]
        if len(self.target_shape) != 3 or self.target_shape[:2] != (h, w) or self.target_shape[2] not in (1, 3):
            raise ValueError("target_shape must be (%d,%d,1) or (%d,%d,3), got %r" % (h, w, h, w, self.target_shape))

    def _tensor_names(self, lib):
        n = getattr(lib, self._API["num_tensors"])()
        return [getattr(lib, self._API["tensor_name"])(i).decode() for i in range(n)]

    def _query_layout(self, lib, offs, sizes, shapes, total):
        spec = self._config(1)
        _lib.check(lib.cpb_vae_spec_layout(C.byref(spec), offs, sizes, shapes, C.byref(total)), "cpb_vae_spec_layout")

    def _workspace_need(self, batch, mode):
        # on this instance's device: the size query initialises the library there (the plan depends on the kernel family)
        spec = self._config(batch)
        with self._on_device():
            return self._libh.cpb_vae_spec_workspace_bytes(C.byref(spec), mode)

    def _initial_weights(self) -> Dict[str, np.ndarray]:
        rng = np.random.RandomState(self._seed if self._seed is not None else np.random.randint(0, 2 ** 31 - 1))
        out = {}
        for name in self._names:
            shape = self._shapes[name]
            if name.endswith("bias"):
                out[name] = np.zeros(shape, np.float32)
                continue
            if len(shape) == 4:
                rf = shape[0] * shape[1]
                fan_in, fan_out = (shape[3] * rf, shape[2] * rf) if "deconv" in name else (shape[2] * rf, shape[3] * rf)
            else:
                fan_in, fan_out = shape
            limit = np.sqrt(6.0 / (fan_in + fan_out))
            out[name] = rng.uniform(-limit, limit, size=shape).astype(np.float32)
        return out

    def _init_logging(self):
        try:
            from torch.utils.tensorboard import SummaryWriter
            self.train_writer = SummaryWriter(os.path.join(self.log_dir, "train"))
            self.val_writer = SummaryWriter(os.path.join(self.log_dir, "val"))
        except Exception as e:   # tensorboard missing: logging is optional, the numerics are not
            print("carla_ppo_b200: TensorBoard logging disabled (%s)" % e)
            self.train_writer = self.val_writer = None

    def _require_session(self):
        if self.sess is None:
            raise CpbError("init_session() has not been called")

    def _on_device(self):
        """Context manager making this model's device current: the C library launches on the CURRENT CUDA device and the
        buffers live on self._device (a model built with device=cuda:1 must work while cuda:0 is current)."""
        return self._torch.cuda.device(self._device)

    def _stream(self):
        return _lib.current_stream_handle(self._device)

    def _call(self, name, *args):
        with self._on_device():
            return _lib.check(getattr(self._libh, name)(*args), name)

    def _broadcast_state(self):
        """data_parallel: every rank adopts rank 0's parameters and optimiser state (different seeds, or a checkpoint only
        rank 0 has, would otherwise train divergent replicas with summed gradients and no error)."""
        world, dist = self._world()
        if world == 1:
            return
        bufs = [self.params]
        if self.training:
            bufs += [self.adam_m, self.adam_v, self.adam_powers]
        for b in bufs:
            dist.broadcast(b, 0)

    # ------------------------------------------------------------------ weights in / out
    def set_weights(self, weights: Dict[str, np.ndarray], adam_m=None, adam_v=None, powers=None):
        """weights: {TF variable name without the ``vae/`` scope: array in the TF layout}."""
        torch = self._torch
        host = np.zeros(self._total, np.float32)
        for name in self._names:
            w = np.asarray(weights[name], np.float32)
            if tuple(w.shape) != self._shapes[name]:
                raise ValueError("%s: expected shape %r, got %r" % (name, self._shapes[name], w.shape))
            o = self._offsets[name]
            host[o:o + w.size] = w.ravel()
        self.params.copy_(torch.from_numpy(host))
        if self.training:
            for buf, src in ((self.adam_m, adam_m), (self.adam_v, adam_v)):
                h = np.zeros(self._total, np.float32)
                if src is not None:
                    for name in self._names:
                        o = self._offsets[name]
                        a = np.asarray(src[name], np.float32)
                        h[o:o + a.size] = a.ravel()
                buf.copy_(torch.from_numpy(h))
            p = (ADAM_BETA1, ADAM_BETA2) if powers is None else powers
            self.adam_powers.copy_(torch.tensor([float(p[0]), float(p[1])], dtype=torch.float32))
        if self.data_parallel:
            self._broadcast_state()

    def _unflatten(self, flat_tensor) -> Dict[str, np.ndarray]:
        host = flat_tensor.detach().cpu().numpy()
        out = {}
        for name in self._names:
            o = self._offsets[name]
            shape = self._shapes[name]
            out[name] = host[o:o + int(np.prod(shape))].reshape(shape).copy()
        return out

    def get_weights(self) -> Dict[str, np.ndarray]:
        self._require_session()
        return self._unflatten(self.params)

    def get_grads(self) -> Dict[str, np.ndarray]:
        return self._unflatten(self.grads)

    # ------------------------------------------------------------------ checkpoints
    def save(self, tf_format=False):
        """One .npz per checkpoint + the text ``checkpoint`` state file tf.train.Saver keeps (max_to_keep=5) under
        the reference's directory layout (vae/models.py:172-175).  ``tf_format=True`` writes the SAME variables as a
        TF-V2 tensor bundle (``model.ckpt-N.index`` / ``.data-00000-of-00001``, tf_bundle.write_bundle) instead, which
        the reference's own ``saver.restore`` reads."""
        self._require_session()
        step = int(self.step_idx)
        prefix = os.path.join(self.checkpoint_dir, "model.ckpt-%d" % step)
        blob = {"vae/" + k: v for k, v in self.get_weights().items()}
        if self.training:
            for k, v in self._unflatten(self.adam_m).items():
                blob["vae/vae/%s/Adam" % k] = v
            for k, v in self._unflatten(self.adam_v).items():
                blob["vae/vae/%s/Adam_1" % k] = v
            pw = self.adam_powers.cpu().numpy()
            blob["vae/beta1_power"], blob["vae/beta2_power"] = pw[0], pw[1]
        blob["vae/step_idx"] = np.int32(step)
        if tf_format:
            from ..tf_bundle import write_bundle
            write_bundle(prefix, {k: np.asarray(v) for k, v in blob.items()})
        else:
            # the frame size the model was built for: load_vae rebuilds it from the checkpoint alone
            blob["vae/source_shape"] = np.asarray(self.source_shape, np.int32)
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
        kept = kept[-5:]
        with open(state, "w") as f:
            f.write('model_checkpoint_path: "%s"\n' % name)
            for k in kept:
                f.write('all_model_checkpoint_paths: "%s"\n' % k)
        print("Model checkpoint saved to {}".format(prefix))

    def load_latest_checkpoint(self):
        """True on success, False when restoring raised, None when there is no checkpoint
        (the reference's three-valued contract, vae/models.py:177-186).  Reads both this build's .npz
        checkpoints and the reference's shipped TF-V2 bundles."""
        self._require_session()
        from ..tf_bundle import BundleReader
        state = os.path.join(self.checkpoint_dir, "checkpoint")
        if not os.path.isfile(state):
            return None
        with open(state) as f:
            m = re.search(r'^model_checkpoint_path:\s*"(.*)"', f.read(), re.M)
        if not m:
            return None
        prefix = m.group(1)
        if not os.path.isabs(prefix):
            prefix = os.path.join(self.checkpoint_dir, prefix)
        try:
            if os.path.isfile(prefix + ".npz"):
                blob = dict(np.load(prefix + ".npz"))
            elif os.path.isfile(prefix + ".index"):
                blob = BundleReader(prefix).all()
            else:
                return None
            recorded = tuple(int(v) for v in blob["vae/source_shape"]) if "vae/source_shape" in blob else None
            if recorded is not None and recorded != self.source_shape:
                raise ValueError("checkpoint %s was written by a model with source_shape %r, this one has %r"
                                 % (prefix, recorded, self.source_shape))
            weights = {n: blob["vae/" + n] for n in self._names}
            m_, v_, pw = None, None, None
            if self.training and ("vae/vae/%s/Adam" % self._names[0]) in blob:
                m_ = {n: blob["vae/vae/%s/Adam" % n] for n in self._names}
                v_ = {n: blob["vae/vae/%s/Adam_1" % n] for n in self._names}
                pw = (float(blob["vae/beta1_power"]), float(blob["vae/beta2_power"]))
            self.set_weights(weights, m_, v_, pw)
            self.step_idx = int(blob["vae/step_idx"]) if "vae/step_idx" in blob else 0
            print("Model checkpoint restored from {}".format(prefix))
            return True
        except Exception as e:
            print(e)
            return False

    # ------------------------------------------------------------------ plumbing
    def _workspace(self, batch, mode):
        key = mode
        need = self._workspace_need(batch, mode)
        _lib.check(need, "workspace_bytes")
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            self._ws[key] = None
            ws = self._torch.empty(int(need), dtype=self._torch.uint8, device=self._device)
            self._ws[key] = ws
        return ws

    def _base_config(self, batch, source_dtype=_lib.FRAME_F32, target_dtype=_lib.FRAME_F32, loss_scale=1.0):
        tscale = 1.0 / 255.0 if self.target_shape[2] == 3 else 1.0 / 12.0
        return VaeConfig(batch, self.target_shape[2], self.z_dim, self.loss_type, source_dtype, target_dtype,
                         tscale, self.beta, self.kl_tolerance, loss_scale)

    def _config(self, batch, source_dtype=_lib.FRAME_F32, target_dtype=_lib.FRAME_F32, loss_scale=1.0):
        """The VaeSpec of the cpb_vae_spec_* entry points: the config at this model's frame size."""
        return VaeSpec(self._base_config(batch, source_dtype, target_dtype, loss_scale), *self.source_shape[:2])

    def _frame_shape(self, channels):
        return tuple(self.source_shape[:2]) + (channels,)

    def _to_device_frames(self, frames, channels):
        """numpy / list / torch -> contiguous CUDA tensor [B,H,W,channels] (source_shape's H, W), float32 or uint8."""
        torch = self._torch
        if not isinstance(frames, torch.Tensor):
            arr = np.asarray(frames)
            if arr.dtype != np.uint8:
                arr = arr.astype(np.float32, copy=False)
            frames = torch.from_numpy(np.ascontiguousarray(arr))
        if frames.dtype not in (torch.float32, torch.uint8):
            frames = frames.to(torch.float32)
        if frames.dim() == 3:
            frames = frames.unsqueeze(0)
        if tuple(frames.shape[1:]) != self._frame_shape(channels):
            raise ValueError("expected frames of shape [B,%d,%d,%d], got %r" % (self._frame_shape(channels) + (tuple(frames.shape),)))
        return frames.to(self._device, non_blocking=True).contiguous()

    @staticmethod
    def _frame_dtype(t):
        return _lib.FRAME_U8 if str(t.dtype).endswith("uint8") else _lib.FRAME_F32

    def _check_flags(self):
        f = int(self._flags.item())
        self._flags.zero_()
        if f & 1:
            raise ValueError("verify_range: source_states outside [0, 1] (reference vae/models.py:24-30, 89)")
        if f & 2:
            raise ValueError("verify_range: target_states outside [0, 1] (reference vae/models.py:24-30, 90)")

    def _eps(self, batch):
        """Standard-normal draws for `batch` rows of THIS rank.  data_parallel: every rank holds the same generator state
        (same seed), draws the noise of the whole global batch and keeps its own contiguous rows -- so the global batch
        sees world*batch independent rows, exactly the rows the single-GPU step would draw for the same seed."""
        torch = self._torch
        world, dist = self._world()
        if world == 1:
            return torch.randn(batch, self.z_dim, generator=self._noise_gen, device=self._device, dtype=torch.float32)
        return dp_noise_rows(torch, self._noise_gen, batch, self.z_dim, dist.get_rank(), world, self._device)

    # ------------------------------------------------------------------ inference surface
    def encode(self, source_states):
        """-> np.float32 [B, z_dim]: the MEAN head (deterministic), vae/models.py:199-202."""
        self._require_session()
        x = self._to_device_frames(source_states, 3)
        return self.encode_device(x).cpu().numpy()

    def encode_device(self, x, return_logvar=False, check=True):
        torch = self._torch
        b = x.shape[0]
        mean = torch.empty(b, self.z_dim, dtype=torch.float32, device=self._device)
        logvar = torch.empty_like(mean) if return_logvar else None
        ws = self._workspace(b, _lib.WS_ENCODE)
        cfg = self._config(b, self._frame_dtype(x))
        self._call(self._API["encode"], C.byref(cfg), _lib.ptr(self.params), _lib.ptr(x), _lib.ptr(mean),
                                             _lib.ptr(logvar), _lib.ptr(self._flags), _lib.ptr(ws), ws.numel(),
                                             self._stream())
        if check:
            self._check_flags()
        return (mean, logvar) if return_logvar else mean

    def generate_from_latent(self, z):
        """-> np.float32 [B, H*W*Ct]: sigmoid of the decoder output, flattened (vae/models.py:188-191)."""
        self._require_session()
        torch = self._torch
        zt = torch.as_tensor(np.asarray(z, np.float32) if not isinstance(z, torch.Tensor) else z,
                             dtype=torch.float32, device=self._device).reshape(-1, self.z_dim).contiguous()
        b = zt.shape[0]
        out = torch.empty(b, int(np.prod(self.target_shape)), dtype=torch.float32, device=self._device)
        ws = self._workspace(b, _lib.WS_FORWARD)
        cfg = self._config(b)
        self._call(self._API["decode"], C.byref(cfg), _lib.ptr(self.params), _lib.ptr(zt), _lib.ptr(out),
                                             _lib.ptr(ws), ws.numel(), self._stream())
        return out.cpu().numpy()

    decode = generate_from_latent

    def reconstruct(self, source_states):
        """-> list of arrays reshaped to source_shape (vae/models.py:193-197).  Runs the same graph the
        reference runs: z is sampled when training=True, the mean otherwise."""
        self._require_session()
        x = self._to_device_frames(source_states, 3)
        out = self.forward_device(x, x if self.target_shape[2] == 3 else None,
                                  eps=self._eps(x.shape[0]) if self.training else None, want_reconstruction=True)
        rec = out["reconstruction"].cpu().numpy()
        return [s.reshape(self.source_shape) for s in rec]

    def forward_device(self, x, y=None, eps=None, want_reconstruction=False, want_latents=False, loss_scale=1.0):
        """The training graph without the optimiser on device tensors.  Returns a dict of device tensors:
        losses[2] (+ mean, logvar, z, reconstruction when requested).  ``y=None`` evaluates against a
        zero target (only meaningful together with want_reconstruction)."""
        torch = self._torch
        b = x.shape[0]
        if y is None:
            y = torch.zeros((b,) + self.target_shape, dtype=torch.float32, device=self._device)
        losses = torch.empty(2, dtype=torch.float32, device=self._device)
        mean = logvar = z = rec = None
        if want_latents:
            mean = torch.empty(b, self.z_dim, dtype=torch.float32, device=self._device)
            logvar = torch.empty_like(mean)
            z = torch.empty_like(mean)
        if want_reconstruction:
            rec = torch.empty(b, int(np.prod(self.target_shape)), dtype=torch.float32, device=self._device)
        ws = self._workspace(b, _lib.WS_FORWARD)
        cfg = self._config(b, self._frame_dtype(x), self._frame_dtype(y), loss_scale)
        self._call(self._API["forward"], C.byref(cfg), _lib.ptr(self.params), _lib.ptr(x), _lib.ptr(y),
                                              _lib.ptr(eps), _lib.ptr(losses), _lib.ptr(mean), _lib.ptr(logvar),
                                              _lib.ptr(z), _lib.ptr(rec), _lib.ptr(self._flags), _lib.ptr(ws),
                                              ws.numel(), self._stream())
        return dict(losses=losses, mean=mean, logvar=logvar, z=z, reconstruction=rec)

    def get_step_idx(self):
        return int(self.step_idx)

    # ------------------------------------------------------------------ training surface
    @property
    def learning_rate(self):
        """The value the reference LOGS (exponential_decay, vae/models.py:140); its Adam uses the constant."""
        return self.base_learning_rate * self.lr_decay ** int(self.step_idx)

    def _world(self):
        if not self.data_parallel:
            return 1, None
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            raise CpbError("data_parallel=True needs an initialised torch.distributed process group")
        return dist.get_world_size(), dist

    def loss_grad_device(self, x, y, eps, loss_scale=1.0):
        """Forward + backward into self.grads / self._losses (device, no sync)."""
        b = x.shape[0]
        ws = self._workspace(b, _lib.WS_TRAIN)
        cfg = self._config(b, self._frame_dtype(x), self._frame_dtype(y), loss_scale)
        self._call(self._API["loss_grad"], C.byref(cfg), _lib.ptr(self.params), _lib.ptr(x), _lib.ptr(y),
                                                _lib.ptr(eps), _lib.ptr(self.grads), _lib.ptr(self._losses),
                                                _lib.ptr(self._flags), _lib.ptr(ws), ws.numel(),
                                                self._stream())

    def adam_device(self, guard=None):
        """TF ApplyAdam on the flat buffers.  ``guard``: device word (tensor) that vetoes the update when non-zero --
        the verify_range flag, so that an out-of-range batch leaves the model untouched like the reference's tf.Assert."""
        self._call("cpb_adam_apply_guarded", _lib.ptr(self.params), _lib.ptr(self.grads), _lib.ptr(self.adam_m),
                   _lib.ptr(self.adam_v), self._total, _lib.ptr(self.adam_powers), self.base_learning_rate, None,
                   ADAM_BETA1, ADAM_BETA2, ADAM_EPS, _lib.ptr(guard), self._stream())

    def train_step_device(self, x, y, eps=None):
        """One minibatch step on device tensors (this rank's shard when data_parallel).  Returns the device
        tensor [recon, kl] of the GLOBAL batch; no host synchronisation."""
        if not self.training:
            raise CpbError("this VAE was built with training=False")
        if eps is None:
            eps = self._eps(x.shape[0])
        world, dist = self._world()
        self.loss_grad_device(x, y, eps, 1.0 / world)
        guard = self._flags
        if world > 1:
            # ONE NCCL all-reduce: flat gradient + the two loss scalars + the verify_range flag (as a float: the sum is
            # non-zero on every rank when ANY rank saw an out-of-range value, so all replicas skip the update together)
            guard = self._gradbuf[self._total + 2:self._total + 3]
            guard.copy_(self._flags)
            dist.all_reduce(self._gradbuf)
        self.adam_device(guard)
        return self._losses

    def train_step(self, source, target, eps=None):
        """One reference minibatch step fed with HOST arrays (the feed_dict of vae/models.py:213-216) through
        cpb_vae_train_step_host.  Returns (recon, kl) floats."""
        self._require_session()
        if not self.training:
            raise CpbError("this VAE was built with training=False")
        torch = self._torch
        world, _ = self._world()
        if world > 1 or isinstance(source, torch.Tensor) or not self._HOST_STEP:
            x = self._to_device_frames(source, 3)
            y = x if target is source else self._to_device_frames(target, self.target_shape[2])
            e = None if eps is None else torch.as_tensor(np.asarray(eps, np.float32), device=self._device)
            losses = self.train_step_device(x, y, e).cpu().numpy()
            self._check_flags()
            return float(losses[0]), float(losses[1])
        src = np.ascontiguousarray(source if np.asarray(source).dtype == np.uint8 else np.asarray(source, np.float32))
        same = target is source
        tgt = src if same else np.ascontiguousarray(target if np.asarray(target).dtype == np.uint8 else np.asarray(target, np.float32))
        b = src.shape[0]
        if eps is None:
            eps = self._eps(b).cpu().numpy()
        eps = np.ascontiguousarray(eps, np.float32)
        sd = _lib.FRAME_U8 if src.dtype == np.uint8 else _lib.FRAME_F32
        td = _lib.FRAME_U8 if tgt.dtype == np.uint8 else _lib.FRAME_F32
        cfg = self._config(b, sd, td)
        need = self._libh.cpb_vae_spec_staging_bytes(C.byref(cfg))
        _lib.check(need, "cpb_vae_spec_staging_bytes")
        st = self._ws.get("staging")
        if st is None or st.numel() < need:
            st = self._ws["staging"] = torch.empty(int(need), dtype=torch.uint8, device=self._device)
        ws = self._workspace(b, _lib.WS_TRAIN)
        losses = np.zeros(2, np.float32)
        flags = np.zeros(1, np.int32)
        self._call("cpb_vae_spec_train_step_host",
            C.byref(cfg), _lib.ptr(self.params), _lib.ptr(self.grads), _lib.ptr(self.adam_m), _lib.ptr(self.adam_v),
            _lib.ptr(self.adam_powers), self.base_learning_rate, _lib.ptr(src), _lib.ptr(src if same else tgt),
            _lib.ptr(eps), _lib.ptr(losses), _lib.ptr(flags), _lib.ptr(st), st.numel(), _lib.ptr(ws), ws.numel(),
            self._stream())
        if flags[0] & 1:
            raise ValueError("verify_range: source_states outside [0, 1]")
        if flags[0] & 2:
            raise ValueError("verify_range: target_states outside [0, 1]")
        return float(losses[0]), float(losses[1])

    class _PendingStep:
        """Handle of a pipelined host-fed step: ``result()`` waits for it and returns (recon, kl)."""

        def __init__(self, vae, slot):
            self._vae, self._slot = vae, slot

        def result(self):
            st = self._vae._pipe
            st["done"][self._slot].synchronize()
            host = st["losses_host"][self._slot]
            if int(host[2]) & 1:
                raise ValueError("verify_range: source_states outside [0, 1]")
            if int(host[2]) & 2:
                raise ValueError("verify_range: target_states outside [0, 1]")
            return float(host[0]), float(host[1])

    def train_step_async(self, source, target=None, eps=None):
        """Host-fed minibatch step with input prefetch: the H2D copy of THIS batch runs on a copy stream (two
        device staging slots) while the previous step still computes; the step is enqueued behind it and the
        losses come back through a pinned buffer.  Returns a handle; call ``.result()`` (typically one step
        later) for (recon, kl).  ``source``/``target`` are host arrays or pinned CPU tensors (fp32 or uint8);
        ``target=None`` or ``target is source`` means the rgb target == source."""
        self._require_session()
        torch = self._torch
        if not self.training:
            raise CpbError("this VAE was built with training=False")

        def as_cpu_tensor(a, channels):
            if not isinstance(a, torch.Tensor):
                arr = np.asarray(a)
                if arr.dtype != np.uint8:
                    arr = arr.astype(np.float32, copy=False)
                a = torch.from_numpy(np.ascontiguousarray(arr))
            if tuple(a.shape[1:]) != self._frame_shape(channels):
                raise ValueError("expected frames of shape [B,%d,%d,%d], got %r" % (self._frame_shape(channels) + (tuple(a.shape),)))
            return a
        same = target is None or target is source
        xs = as_cpu_tensor(source, 3)
        ys = xs if same else as_cpu_tensor(target, self.target_shape[2])
        b = xs.shape[0]
        key = (b, xs.dtype, ys.dtype, same)
        st = getattr(self, "_pipe", None)
        if st is None or st["key"] != key:
            dev = self._device
            st = self._pipe = {
                "key": key, "i": 0, "copy_stream": torch.cuda.Stream(device=dev),
                "x": [torch.empty((b,) + self.source_shape, dtype=xs.dtype, device=dev) for _ in range(2)],
                "y": [None, None] if same else [torch.empty((b,) + self.target_shape, dtype=ys.dtype, device=dev) for _ in range(2)],
                "eps": [torch.empty((b, self.z_dim), dtype=torch.float32, device=dev) for _ in range(2)],
                "copied": [torch.cuda.Event() for _ in range(2)], "done": [torch.cuda.Event() for _ in range(2)],
                "used": [False, False],
                "losses_dev": [torch.zeros(3, dtype=torch.float32, device=dev) for _ in range(2)],
                "losses_host": [torch.zeros(3, dtype=torch.float32).pin_memory() for _ in range(2)],
            }
        slot = st["i"] % 2
        st["i"] += 1
        compute = torch.cuda.current_stream()
        cs = st["copy_stream"]
        if st["used"][slot]:
            cs.wait_event(st["done"][slot])            # the step that last read this slot has finished
        with torch.cuda.stream(cs):
            st["x"][slot].copy_(xs, non_blocking=True)
            if not same:
                st["y"][slot].copy_(ys, non_blocking=True)
            if eps is not None:
                e = eps if isinstance(eps, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(eps, np.float32))
                st["eps"][slot].copy_(e, non_blocking=True)
            st["copied"][slot].record(cs)
        compute.wait_event(st["copied"][slot])
        if eps is None:
            st["eps"][slot].copy_(self._eps(b))
        x = st["x"][slot]
        y = x if same else st["y"][slot]
        losses = self.train_step_device(x, y, st["eps"][slot])
        ld = st["losses_dev"][slot]
        ld[:2].copy_(losses)
        ld[2:3].copy_(self._flags.to(torch.float32))
        self._flags.zero_()
        st["losses_host"][slot].copy_(ld, non_blocking=True)
        st["done"][slot].record(compute)
        st["used"][slot] = True
        return VAE._PendingStep(self, slot)

    def _device_dataset(self, arr, channels):
        """Upload a host dataset once and keep it resident (keyed on the array's identity and buffer)."""
        torch = self._torch
        if isinstance(arr, torch.Tensor):
            return self._to_device_frames(arr, channels)
        a = np.asarray(arr)
        key = (id(arr), a.__array_interface__["data"][0], a.shape, str(a.dtype))
        # content fingerprint: ~64 K values sampled at a fixed stride over the whole array.  The reference re-feeds host
        # data every step; a caller that rewrites the array in place between epochs (augmentation, buffer reuse) must not
        # silently train on the stale GPU copy.  (Edits that miss every sampled value are not detected: call
        # clear_dataset_cache(), or pass resident_dataset=False to the constructor to upload on every epoch.)
        flat = a.reshape(-1)
        probe = flat[::max(1, flat.size // 65536)]
        finger = (float(probe.astype(np.float64).sum()), float(probe[::7].astype(np.float64).sum()))
        hit = self._dataset_cache.get(key)
        if hit is None or hit[1] != finger or not self._resident_dataset:
            if len(self._dataset_cache) >= 4:
                self._dataset_cache.clear()
            hit = self._dataset_cache[key] = (self._to_device_frames(a, channels), finger)
        return hit[0]

    def clear_dataset_cache(self):
        self._dataset_cache.clear()

    def _epoch(self, source, target, batch_size, train):
        torch = self._torch
        n = len(source)
        world, dist = self._world()
        xs = self._device_dataset(source, 3)
        ys = xs if target is source else self._device_dataset(target, self.target_shape[2])
        indices = np.arange(n)
        np.random.shuffle(indices)                      # same host RNG call as the reference (:208-209)
        if world > 1:                                   # one shuffle for the whole job: rank 0's (ranks seed np.random independently)
            indices = dp_shared_permutation(torch, dist, indices, self._device)
        steps = n // batch_size                         # tail N % B dropped like the reference (:211)
        rank = dist.get_rank() if world > 1 else 0
        shard = batch_size // world
        if world > 1 and batch_size % world != 0:
            raise ValueError("batch_size must be divisible by the world size")
        idx_dev = torch.from_numpy(indices[:steps * batch_size].astype(np.int64)).to(self._device)
        acc = torch.zeros(2, dtype=torch.float64, device=self._device)
        for i in range(steps):
            mb = idx_dev[i * batch_size + rank * shard:i * batch_size + (rank + 1) * shard]
            x = xs.index_select(0, mb)
            y = x if ys is xs else ys.index_select(0, mb)
            if train:
                losses = self.train_step_device(x, y)
            else:
                eps = self._eps(x.shape[0]) if self.training else None
                losses = self.forward_device(x, y, eps, loss_scale=1.0 / world)["losses"]
                if world > 1:
                    dist.all_reduce(losses)
            acc += losses.double()
        self._check_flags()
        mean = (acc / max(steps, 1)).cpu().numpy()      # tf.metrics.mean over the minibatch means
        self._last_metrics = (float(mean[0]), float(mean[1]))
        return self._last_metrics

    def train_one_epoch(self, train_source, train_target, batch_size):
        self._require_session()
        if not self.training:
            raise CpbError("this VAE was built with training=False")
        recon, kl = self._epoch(train_source, train_target, batch_size, True)
        self._write_summary(self.train_writer, recon, kl)
        self.step_idx += 1                              # step_idx counts EPOCHS (vae/models.py:218)

    def evaluate(self, val_source, val_target, batch_size):
        self._require_session()
        recon, kl = self._epoch(val_source, val_target, batch_size, False)
        self._write_summary(self.val_writer, recon, kl)
        return [recon, kl]

    def _write_summary(self, writer, recon, kl):
        if writer is None:
            return
        step = self.get_step_idx()
        writer.add_scalar("vae/kl_loss", kl, step)
        writer.add_scalar("vae/reconstruction_loss", recon, step)
        writer.add_scalar("vae/learning_rate", self.learning_rate, step)
        writer.flush()


class ConvVAE(VAE):
    """Convolutional VAE (reference vae/models.py:233-268) at any frame size the reference builds: source_shape (H, W, 3)
    with H and W multiples of 16 in [48, 512] (80x160 in the reference's own data), target_shape (H, W, 1 or 3); the
    target defaults to the source at 80x160 only.  encoded_shape is (H/16 - 2, W/16 - 2, 256)."""

    def __init__(self, source_shape, target_shape=None, **kwargs):
        if target_shape is None:
            # target_shape defaults to source_shape (an rgb target) at the reference's 80x160 only; a model built for
            # another frame size names its target, (H, W, 3) or (H, W, 1), as train_vae.py and load_vae do
            h, w = (int(v) for v in tuple(source_shape)[:2])
            if (h, w) != (80, 160):
                raise ValueError(frame_rule_error(h, w) or "ConvVAE at frame %dx%d: give target_shape, (%d, %d, 3) for an rgb "
                                 "target or (%d, %d, 1) for a segmentation target" % (h, w, h, w, h, w))
            target_shape = source_shape
        super().__init__(source_shape, target_shape, None, None, **kwargs)


class MlpVAE(VAE):
    """The reference's dense VAE (vae/models.py:271-299): flatten -> one dense relu layer per encoder size -> mean /
    logstd_sqare -> sample -> one dense relu layer per decoder size -> dense(prod(target_shape)) = logits.  Same surface
    as ConvVAE.  Each side takes 1 to 8 hidden sizes, each a multiple of 32 in [32, 8192]; the variables carry the
    reference's names (encoder/dense, encoder/dense_1, ..., decoder/dense_M for the output layer).  The dense layers run
    on the fp32 SIMT kernels of the library (cpb_mlpvae_spec_* entry points) in math modes 0 and 1.  In math mode 2
    (cpb_set_math_mode(2), ``train_vae.py --math_mode tf32``) the five frame-wide products -- the first encoder layer's
    forward and weight gradient, the output layer's forward, data gradient and weight gradient -- run as one TF32
    tensor-core pass with both operands rounded to nearest (not fp32-accurate); the rest runs as in mode 1.  The
    workspace is re-sized on every call, so switching the mode between calls is safe."""

    _API = {"encode": "cpb_mlpvae_spec_encode", "decode": "cpb_mlpvae_spec_decode", "forward": "cpb_mlpvae_spec_forward",
            "loss_grad": "cpb_mlpvae_spec_loss_grad", "encode_predict": "cpb_mlpvae_encode_predict"}
    _HOST_STEP = False

    def __init__(self, source_shape, target_shape=None, encoder_sizes=(512, 256), decoder_sizes=(256, 512), **kwargs):
        target_shape = source_shape if target_shape is None else target_shape
        self.encoder_sizes = tuple(int(v) for v in encoder_sizes)
        self.decoder_sizes = tuple(int(v) for v in decoder_sizes)
        for name, sizes in (("encoder_sizes", self.encoder_sizes), ("decoder_sizes", self.decoder_sizes)):
            if not 1 <= len(sizes) <= _lib.MLP_MAX_LAYERS or any(v < 32 or v > 8192 or v % 32 for v in sizes):
                raise ValueError("MlpVAE %s must hold 1 to %d sizes, each a multiple of 32 in [32, 8192], got %r"
                                 % (name, _lib.MLP_MAX_LAYERS, sizes))
        super().__init__(source_shape, target_shape, None, None, **kwargs)
        self.encoded_shape = (self.encoder_sizes[-1],)

    def _check_shapes(self):
        if self.source_shape != (80, 160, 3):
            raise ValueError("MlpVAE is built for source_shape (80,160,3) (reference vae/models.py:243-244), got %r"
                             % (self.source_shape,))
        if self.target_shape[:2] != (80, 160) or self.target_shape[2] not in (1, 3):
            raise ValueError("target_shape must be (80,160,1) or (80,160,3), got %r" % (self.target_shape,))

    def _spec(self, batch, source_dtype=_lib.FRAME_F32, target_dtype=_lib.FRAME_F32, loss_scale=1.0):
        base = self._base_config(batch, source_dtype, target_dtype, loss_scale)
        return MlpVaeSpec.of(base, self.encoder_sizes, self.decoder_sizes)

    _config = _spec

    def _mlp_config(self, batch, source_dtype=_lib.FRAME_F32, target_dtype=_lib.FRAME_F32, loss_scale=1.0):
        """The two-per-side MlpVaeConfig of the cpb_mlpvae_* entry points; only a model with two hidden layers per
        side has one."""
        if len(self.encoder_sizes) != 2 or len(self.decoder_sizes) != 2:
            raise ValueError("MlpVaeConfig describes two hidden layers per side; this model has %d and %d"
                             % (len(self.encoder_sizes), len(self.decoder_sizes)))
        base = self._base_config(batch, source_dtype, target_dtype, loss_scale)
        return MlpVaeConfig(base, self.encoder_sizes[0], self.encoder_sizes[1], self.decoder_sizes[0], self.decoder_sizes[1])

    def _tensor_names(self, lib):
        spec = self._spec(1)
        n = _lib.check(lib.cpb_mlpvae_spec_num_tensors(C.byref(spec)), "cpb_mlpvae_spec_num_tensors")
        return [lib.cpb_mlpvae_spec_tensor_name(C.byref(spec), i).decode() for i in range(n)]

    def _query_layout(self, lib, offs, sizes, shapes, total):
        spec = self._spec(1)
        _lib.check(lib.cpb_mlpvae_spec_layout(C.byref(spec), offs, sizes, shapes, C.byref(total)), "cpb_mlpvae_spec_layout")

    def _workspace_need(self, batch, mode):
        spec = self._spec(batch)
        return self._libh.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), mode)
