"""The harness the tests of the library share: loading it, its process-global state, the two VAE constructors, and the
readers of their workspaces.

Test modules import the fixtures by name (`from harness import lib, library_state`): a fixture imported into a module
applies to that module, autouse ones included."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from helpers import rel_l2


@pytest.fixture(scope="module")
def lib():
    """The library, built first when a clean checkout has no build of it."""
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(autouse=True)
def library_state(lib):
    """The library's state outlives a test: after each one the whole backward pass runs again, in math mode 1."""
    yield
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_debug_vae_backward_stop(None))
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_3XTF32))


@pytest.fixture
def fp32_matmul():
    """torch's CUDA matmuls in plain fp32 for the test (the err_f32 references), restored after it."""
    import torch
    allow = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = allow


@contextlib.contextmanager
def math_mode(lib, mode):
    """Math `mode` inside the block, the mode before it after."""
    from carla_ppo_b200 import _lib
    old = lib.cpb_get_math_mode()
    _lib.check(lib.cpb_set_math_mode(mode))
    try:
        yield
    finally:
        _lib.check(lib.cpb_set_math_mode(old))


def gate(approx, ref, floor):
    """The parity gate: max(floor, 2 x the distance of the restatement `approx` from the float64 `ref`)."""
    return max(floor, 2.0 * rel_l2(approx, ref))


def dev(vae, a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device=vae._device)


def make_conv_vae(tmp_path, weights=None, hw=(80, 160), ct=3, loss="mse", z=64, tag="m", **kw):
    from carla_ppo_b200.vae.models import ConvVAE
    h, w = hw
    vae = ConvVAE((h, w, 3), target_shape=(h, w, ct), z_dim=z, loss_fn=loss, model_dir=str(tmp_path / tag), seed=0, **kw)
    vae.init_session(init_logging=False)
    if weights is not None:
        vae.set_weights(weights)
    return vae


def make_mlp(tmp_path, weights=None, enc=(512, 256), dec=(256, 512), loss="bce", z=64, ct=3, tag="m", training=True):
    from carla_ppo_b200.vae.models import MlpVAE
    vae = MlpVAE(source_shape=(80, 160, 3), target_shape=(80, 160, ct), z_dim=z, loss_fn=loss, encoder_sizes=enc,
                 decoder_sizes=dec, model_dir=str(tmp_path / ("mlp_zdim%d_%s" % (z, tag))), seed=0, training=training)
    vae.init_session(init_logging=False)
    if weights is not None:
        vae.set_weights(weights)
    return vae


# ----------------------------------------------------------------------------------------------- ConvVAE workspace
CONV_BUFFERS = ["xp", "a1", "a2", "a3", "a4", "heads", "z", "d1", "b1", "b2", "b3", "logits_p", "gA", "gB", "frame_loss",
                "kl_rows", "gz", "gheads"]
RELU_LAYERS = {"a1": "conv1", "a2": "conv2", "a3": "conv3", "a4": "conv4", "b1": "deconv1", "b2": "deconv2",
               "b3": "deconv3"}


def sides(h, w):
    """(H, W) of the frame and of the outputs of conv1-4 (deconv3-1 mirror them)."""
    out = [(h, w)]
    for _ in range(4):
        h, w = (h - 4) // 2 + 1, (w - 4) // 2 + 1
        out.append((h, w))
    return out


def conv_workspace(vae, batch, ws_mode):
    """The buffers of the last call that used workspace `ws_mode`, as float32 device views shaped for the model's frame
    size (a buffer the workspace does not hold is left out).  "g" holds the raw bytes from the start of each ping-pong
    gradient buffer, gA and gB, in the training workspace."""
    import torch
    from carla_ppo_b200 import _lib
    offs = (C.c_int64 * len(CONV_BUFFERS))()
    n = _lib.load().cpb_debug_vae_spec_buffer_offsets(C.byref(vae._config(batch)), ws_mode, offs, len(CONV_BUFFERS))
    assert n == len(CONV_BUFFERS)
    s = sides(*vae.source_shape[:2])
    zp = 64 * ((vae.z_dim + 63) // 64)

    def sh(level, c):
        return (batch,) + s[level] + (c,)
    shapes = {"xp": sh(0, 4), "a1": sh(1, 32), "a2": sh(2, 64), "a3": sh(3, 128), "a4": sh(4, 256), "heads": (2, batch, zp),
              "z": (batch, zp), "d1": sh(4, 256), "b1": sh(3, 128), "b2": sh(2, 64), "b3": sh(1, 32), "logits_p": sh(0, 4),
              "frame_loss": (batch,), "kl_rows": (batch,), "gz": (batch, zp), "gheads": (2, batch, zp)}
    ws = vae._ws[ws_mode]
    out = {}
    for name, o in zip(CONV_BUFFERS, offs):
        if name in shapes and o >= 0:
            out[name] = ws[o:o + 4 * int(np.prod(shapes[name]))].view(torch.float32).view(shapes[name])
    g = dict(zip(CONV_BUFFERS, offs))
    out["g"] = {"gA": ws[g["gA"]:], "gB": ws[g["gB"]:]} if g["gA"] >= 0 else {}
    return out


def conv_relu_masks(vae, batch):
    """The ReLU activity pattern of the last loss_grad call, {layer: bool array}."""
    from carla_ppo_b200 import _lib
    v = conv_workspace(vae, batch, _lib.WS_TRAIN)
    return {layer: v[name].cpu().numpy() > 0 for name, layer in RELU_LAYERS.items()}


# ----------------------------------------------------------------------------------------------- MlpVAE workspace
def mlp_buffer_names(vae):
    return (["x"] + ["h%d" % i for i in range(len(vae.encoder_sizes))] + ["heads", "z"] +
            ["g%d" % j for j in range(len(vae.decoder_sizes))] + ["logits", "ga", "gb"])


def mlp_workspace(vae, batch, ws_mode, widths, frames=None, host=True):
    """Named buffers of the last call that used workspace `ws_mode`, read back from the device as [batch, width] float64
    arrays -- only the rows `frames` when given; host=False: the float32 device views, all rows."""
    import torch
    from carla_ppo_b200 import _lib
    names = mlp_buffer_names(vae)
    offs = (C.c_int64 * len(names))()
    spec = vae._config(batch)
    assert _lib.load().cpb_debug_mlpvae_spec_buffer_offsets(C.byref(spec), ws_mode, offs, len(names)) == len(names)
    ws = vae._ws[ws_mode]
    out = {}
    for nm, width in widths.items():
        o = offs[names.index(nm)]
        t = ws[o:o + 4 * batch * width].view(torch.float32).view(batch, width)
        if host:
            t = (t if frames is None else t[frames]).cpu().numpy().astype(np.float64)
        out[nm] = t
    return out


def mlp_relu_masks(vae, batch, frames=None):
    """The device's ReLU activity pattern of every hidden layer after a loss_grad call (of the rows `frames` if given)."""
    from carla_ppo_b200 import _lib
    widths = {"h%d" % i: v for i, v in enumerate(vae.encoder_sizes)}
    widths.update({"g%d" % j: v for j, v in enumerate(vae.decoder_sizes)})
    return {k: v > 0 for k, v in mlp_workspace(vae, batch, _lib.WS_TRAIN, widths, frames).items()}
