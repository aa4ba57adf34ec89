"""The ConvVAE at frame sizes other than 80x160, on the GPU: end to end against the float64 oracle, every layer pass on the
device's own operands, the legacy 80x160 entry points against their cpb_vae_spec_* twins bit for bit, the tensor-core
batch bound, and the RL path (fused actor, train.py, train_vae.py) at 64x128.

Geometries: 48x48 (the encoder ends on one pixel), 64x96 (H4 and W4 even: the other quad-form parity of conv4's data
gradient and deconv1's forward pass), 96x64, 112x208 (both odd), 48x512 and 512x48 (one-pixel-tall / -wide small
images), 160x320, and 512x512 at B = 2 only."""
import contextlib
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

import test_vae_layers_gpu as L
from helpers import committed_frames, rel_l2

pytestmark = pytest.mark.gpu

GEOMETRIES = [(48, 48), (64, 96), (96, 64), (112, 208), (48, 512), (512, 48), (160, 320), (512, 512)]
CONFIGS = {"rgb-bce-z64": (3, "bce", 64), "seg-mse-z100": (1, "mse", 100)}
FWD_FLOOR, GRAD_FLOOR = 1e-5, 2e-5     # the floors of tests/test_vae_gpu.py


def sides(h, w):
    out = [(h, w)]
    for _ in range(4):
        h, w = (h - 4) // 2 + 1, (w - 4) // 2 + 1
        out.append((h, w))
    return out


@pytest.fixture(scope="module")
def lib():
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(autouse=True)
def restore(lib):
    yield
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_debug_vae_backward_stop(None))
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_3XTF32))


def make_vae(tmp_path, hw, ct=3, loss="mse", z=64, weights=None, tag="m", **kw):
    from carla_ppo_b200.vae.models import ConvVAE
    h, w = hw
    vae = ConvVAE((h, w, 3), target_shape=(h, w, ct), z_dim=z, loss_fn=loss, model_dir=str(tmp_path / tag), seed=0, **kw)
    vae.init_session(init_logging=False)
    if weights is not None:
        vae.set_weights(weights)
    return vae


def dev(vae, a):
    return torch.as_tensor(np.ascontiguousarray(a), device=vae._device)


def spec_masks(lib, vae, batch):
    """The ReLU activity pattern of the last loss_grad call, read back through cpb_debug_vae_spec_buffer_offsets."""
    from carla_ppo_b200 import _lib
    names = ["xp", "a1", "a2", "a3", "a4", "heads", "z", "d1", "b1", "b2", "b3"]
    offs = (C.c_int64 * len(names))()
    spec = vae._config(batch)
    assert lib.cpb_debug_vae_spec_buffer_offsets(C.byref(spec), _lib.WS_TRAIN, offs, len(names)) == len(names)
    s = sides(*vae.source_shape[:2])
    shapes = {"a1": s[1] + (32,), "a2": s[2] + (64,), "a3": s[3] + (128,), "a4": s[4] + (256,),
              "b1": s[3] + (128,), "b2": s[2] + (64,), "b3": s[1] + (32,)}
    layer = {"a1": "conv1", "a2": "conv2", "a3": "conv3", "a4": "conv4", "b1": "deconv1", "b2": "deconv2", "b3": "deconv3"}
    ws = vae._ws[_lib.WS_TRAIN]
    out = {}
    for nm, o in zip(names, offs):
        if nm in shapes:
            cnt = batch * int(np.prod(shapes[nm]))
            out[layer[nm]] = ws[o:o + 4 * cnt].view(torch.float32).cpu().numpy().reshape((batch,) + shapes[nm]) > 0
    return out


# --------------------------------------------------------------------------------------------------- end to end
E2E = [(g, b) for g in GEOMETRIES if g != (512, 512) for b in (1, 3)] + [((512, 512), 2)]


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["simt", "tc3xtf32", "tf32"])
@pytest.mark.parametrize("hw,batch", E2E, ids=["%dx%d-B%d" % (g + (b,)) for g, b in E2E])
def test_end_to_end_against_the_float64_oracle(lib, tmp_path, hw, batch, mode, cfg):
    """mu, logvar, z, the reconstruction, both losses, all 22 gradients (on the device's ReLU masks) and two Adam steps
    against float64, gated at max(floor, 2 x the error of the float32 restatement) -- the TF32 restatement in mode 2."""
    from carla_ppo_b200 import _lib
    from oracle import torch_ref, vae_oracle as vo
    import tf32_oracle
    ct, loss, z = CONFIGS[cfg]
    h, w = hw
    _lib.check(lib.cpb_set_math_mode(mode))
    p = vo.glorot_init(h + w + batch, (h, w, 3), ct, z)
    rs = np.random.RandomState(h * w + batch)
    for k in p:
        if k.endswith("bias"):
            p[k] = (0.05 * rs.randn(*p[k].shape)).astype(np.float32)
    x = rs.rand(batch, h, w, 3).astype(np.float32)
    y = x if ct == 3 else rs.rand(batch, h, w, 1).astype(np.float32)
    eps = rs.randn(batch, z).astype(np.float32)
    vae = make_vae(tmp_path, hw, ct, loss, z, p)

    def restated(masks=None):
        if mode == 2:
            return tf32_oracle.loss_and_grads(p, x, y, eps, loss, relu_masks=masks)
        return torch_ref.vae_loss_and_grads(p, x, y, eps, loss, dtype=torch.float32)

    # forward
    out = vae.forward_device(dev(vae, x), dev(vae, y), dev(vae, eps), want_reconstruction=True, want_latents=True)
    ref = vo.loss_and_grads(p, x, y, eps, loss, want_grads=False)
    r32 = restated()
    for key in ("mean", "logvar", "z"):
        gate = max(FWD_FLOOR, 2 * rel_l2(r32[key], ref[key]))
        assert rel_l2(out[key].cpu().numpy(), ref[key]) < gate, key
    rec = out["reconstruction"].cpu().numpy().reshape(batch, h, w, ct)
    gate = max(FWD_FLOOR, 2 * rel_l2(vo.sigmoid(np.asarray(r32["logits"], np.float64)), vo.sigmoid(ref["logits"])))
    assert rel_l2(rec, vo.sigmoid(ref["logits"])) < gate
    losses = out["losses"].cpu().numpy()
    assert abs(losses[0] - ref["recon"]) < max(FWD_FLOOR, 2 * abs(r32["recon"] - ref["recon"]) / ref["recon"]) * ref["recon"]
    assert abs(losses[1] - ref["kl"]) < max(FWD_FLOOR, 2 * abs(r32["kl"] - ref["kl"]) / max(ref["kl"], 1)) * max(ref["kl"], 1)

    # gradients on the device's ReLU masks
    vae.loss_grad_device(dev(vae, x), dev(vae, y), dev(vae, eps))
    got = vae.get_grads()
    masks = spec_masks(lib, vae, batch)
    g64 = vo.loss_and_grads(p, x, y, eps, loss, relu_masks=masks)
    g32 = restated(masks if mode == 2 else None)
    # the device's ReLU pattern differs from float64's only where the pre-activation is negligible at the mode's precision
    for name, pre in g64["relu_pre"].items():
        flips = masks[name] != (pre > 0)
        if flips.any():
            rms = np.sqrt(np.mean(pre * pre))
            assert np.abs(pre[flips]).max() < (5e-3 if mode == 2 else 2e-5) * rms, (name, np.abs(pre[flips]).max() / rms)
    assert len(got) == 22
    for name, g in g64["grads"].items():
        gate = max(GRAD_FLOOR, 2 * rel_l2(g32["grads"][name], g))
        assert rel_l2(got[name], g) < gate, (name, rel_l2(got[name], g), gate)

    # two Adam steps on the same batch: TF ApplyAdam in float64 on the gradients each step computed (the gradients
    # themselves are gated above; Adam's first steps are ~lr * sign(g), so a ~0 gradient of the other sign moves an
    # element by 2 lr in any fp32 implementation)
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    state = vo.adam_init_state(p64)
    for _ in range(2):
        vae.train_step_device(dev(vae, x), dev(vae, y), dev(vae, eps))
        vo.adam_apply(p64, {k: g.astype(np.float64) for k, g in vae.get_grads().items()}, state, 1e-4)
    after = vae.get_weights()
    for k in p64:
        assert rel_l2(after[k], p64[k]) < 1e-6, k
    assert np.allclose(vae.adam_powers.cpu().numpy(), [0.9 ** 3, 0.999 ** 3], rtol=1e-6)


@pytest.mark.parametrize("hw", [(64, 96), (112, 208), (48, 512)])
def test_uint8_frames_and_verify_range(lib, tmp_path, hw):
    from carla_ppo_b200 import _lib
    h, w = hw
    rs = np.random.RandomState(3)
    u8 = rs.randint(0, 256, size=(3, h, w, 3)).astype(np.uint8)
    vae = make_vae(tmp_path, hw, 3, "bce")
    for mode in (0, 1, 2):
        _lib.check(lib.cpb_set_math_mode(mode))
        a = vae.encode(u8)
        b = vae.encode(u8.astype(np.float32) * np.float32(1.0 / 255.0))    # the loader's own scaling: the same floats
        assert a.shape == (3, 64) and np.array_equal(a, b), mode
    # an out-of-range source sets the flag and leaves the model untouched (the reference's tf.Assert)
    before = vae.params.clone()
    bad = rs.rand(2, h, w, 3).astype(np.float32)
    bad[1, h - 1, w - 1, 2] = 1.5
    with pytest.raises(ValueError, match="verify_range"):
        vae.train_step(bad, bad)
    assert torch.equal(vae.params, before)
    vae.train_step(bad.clip(0, 1), bad.clip(0, 1))
    assert not torch.equal(vae.params, before)


# --------------------------------------------------------------------------------------------------- every layer pass
class GeoCase(L.Case):
    """tests/test_vae_layers_gpu.py's Case at frame size hw: the same passes, gates and stops, shapes from the geometry."""

    def __init__(self, lib, tmp_path, mode, B, ct, z, hw):
        from carla_ppo_b200 import _lib
        from carla_ppo_b200.vae.models import ConvVAE
        from oracle import vae_oracle as vo
        h, w = hw
        self.s = sides(h, w)
        self.lib, self.mode, self.B, self.ct, self.z, self.zp = lib, mode, B, ct, z, 64 * ((z + 63) // 64)
        self.j = L.Judge("%dx%d mode %d B=%d ct=%d z=%d" % (h, w, mode, B, ct, z))
        _lib.check(lib.cpb_set_math_mode(mode))
        wts = vo.glorot_init(B + 10 * ct + h, (h, w, 3), ct, z)
        rs = np.random.RandomState(B + ct + w)
        for k in wts:
            if k.endswith("bias"):
                wts[k] = (0.05 * rs.randn(*wts[k].shape)).astype(np.float32)
        self.vae = ConvVAE((h, w, 3), target_shape=(h, w, ct), z_dim=z, loss_fn="mse" if ct == 3 else "bce",
                           model_dir=str(tmp_path / "m"), seed=0)
        self.vae.init_session(init_logging=False)
        self.vae.set_weights(wts)
        d = self.vae._device
        self.w = {k: torch.from_numpy(v).to(d) for k, v in wts.items()}
        g = torch.Generator(device=d)
        g.manual_seed(1000 + B)
        self.x = torch.rand(B, h, w, 3, generator=g, device=d)
        self.y = self.x if ct == 3 else torch.rand(B, h, w, 1, generator=g, device=d)
        self.eps = torch.randn(B, z, generator=g, device=d)

    def shape(self, level, c):
        return (self.B,) + self.s[level] + (c,)

    @contextlib.contextmanager
    def feat_floor(self):
        """The gate floor of a reduction over the FEAT = H4*W4*256 features (heads forward, dense1's data gradient):
        tests/test_vae_layers_gpu.py's floor holds for FEAT = 6144; the rounding error of a serial fp32 sum grows as the
        square root of its length, so the floor scales by sqrt(FEAT / 6144) above it (x 6.1 at 512x512)."""
        floor = L.FLOOR
        L.FLOOR = floor * max(1.0, np.sqrt(int(np.prod(self.s[4])) * 256 / 6144))
        try:
            yield
        finally:
            L.FLOOR = floor

    def _views(self, ws_mode):
        offs = (C.c_int64 * len(L.BUFFERS))()
        spec = self.vae._config(self.B)
        n = self.lib.cpb_debug_vae_spec_buffer_offsets(C.byref(spec), ws_mode, offs, len(L.BUFFERS))
        assert n == len(L.BUFFERS)
        ws = self.vae._ws[ws_mode]
        B, zp, sh = self.B, self.zp, self.shape
        shapes = {"xp": sh(0, 4), "a1": sh(1, 32), "a2": sh(2, 64), "a3": sh(3, 128), "a4": sh(4, 256), "heads": (2, B, zp),
                  "z": (B, zp), "d1": sh(4, 256), "b1": sh(3, 128), "b2": sh(2, 64), "b3": sh(1, 32), "logits_p": sh(0, 4),
                  "gz": (B, zp), "gheads": (2, B, zp)}
        out = {}
        for name, o in zip(L.BUFFERS, offs):
            if name in shapes and o >= 0:
                out[name] = ws[o:o + 4 * int(np.prod(shapes[name]))].view(torch.float32).view(shapes[name])
        out["g"] = {"gA": ws[offs[L.BUFFERS.index("gA")]:], "gB": ws[offs[L.BUFFERS.index("gB")]:]} if offs[12] >= 0 else {}
        return out

    def forward(self):
        from carla_ppo_b200 import _lib
        self._poisoned(_lib.WS_FORWARD)
        self.vae.forward_device(self.x, self.y, self.eps)
        torch.cuda.synchronize()
        v = self._views(_lib.WS_FORWARD)
        j, B, z, op, wt, s = self.j, self.B, self.z, self._op, self._wt, self.s
        R, relu = L.R, torch.relu

        def conv(name, src, tc):
            def ref(dt, f0, f1):
                a = op(v[src], tc, dt, f0, f1)
                if src == "xp":
                    a = a[..., :3]
                return relu(R.gather(a, wt("encoder/%s/kernel" % name, tc, dt)) + self.w["encoder/%s/bias" % name].to(dt))
            return ref

        def deconv(name, src, tc, out_hw, act=True):
            def ref(dt, f0, f1):
                r = R.scatter(op(v[src], tc, dt, f0, f1), wt("decoder/%s/kernel" % name, tc, dt), out_hw) + \
                    self.w["decoder/%s/bias" % name].to(dt)
                return relu(r) if act else r
            return ref

        L.check_frames(j, "conv1.fwd", v["a1"], conv("conv1", "xp", False), B)
        L.check_frames(j, "conv2.fwd", v["a2"], conv("conv2", "a1", True), B)
        L.check_frames(j, "conv3.fwd", v["a3"], conv("conv3", "a2", True), B)
        L.check_frames(j, "conv4.fwd", v["a4"], conv("conv4", "a3", True), B)
        for i, (kn, bn) in enumerate((("mean/kernel", "mean/bias"), ("logstd_sqare/kernel", "logstd_sqare/bias"))):
            with self.feat_floor():
                L.check_frames(j, "heads.fwd %d" % i, v["heads"][i, :, :z], lambda dt, f0, f1, kn=kn, bn=bn: (
                    op(v["a4"], False, dt, f0, f1).reshape(f1 - f0, -1) @ wt(kn, False, dt) + self.w[bn].to(dt)), B)
        if not bool((v["heads"][:, :, z:] == 0).all()):
            j.failures.append("heads.fwd %s: padded columns are not 0" % j.tag)
        L.check_frames(j, "dense1.fwd", v["d1"], lambda dt, f0, f1: (
            R.dense1_fwd(op(v["z"], False, dt, f0, f1), wt("decoder/dense1/kernel", False, dt))
            + self.w["decoder/dense1/bias"].to(dt)).reshape((f1 - f0,) + s[4] + (256,)), B)
        L.check_frames(j, "deconv1.fwd", v["b1"], deconv("deconv1", "d1", True, s[3]), B)
        L.check_frames(j, "deconv2.fwd", v["b2"], deconv("deconv2", "b1", True, s[2]), B)
        L.check_frames(j, "deconv3.fwd", v["b3"], deconv("deconv3", "b2", True, s[1]), B)
        L.check_frames(j, "deconv4.fwd", v["logits_p"][..., :self.ct], deconv("deconv4", "b3", False, s[0], act=False), B)

    def _group_deconv4(self, v, grads):
        ct, op, wt, R = self.ct, self._op, self._wt, L.R
        dlog = v["logits_p"][..., :ct]
        gA = self._grad_view(v["g"]["gA"], self.shape(1, 32))
        self.j.finite("deconv4 input gradient", dlog)
        self._conv_group(grads, "deconv4", "decoder/deconv4", dlog,
                         lambda dt, f0, f1: (op(dlog, False, dt, f0, f1), op(v["b3"], False, dt, f0, f1)),
                         (gA, lambda dt, f0, f1: R.gather(op(dlog, False, dt, f0, f1), wt("decoder/deconv4/kernel", False, dt))
                          * (v["b3"][f0:f1] > 0)))

    def _group_deconv3(self, v, grads):
        self._deconv_group(v, grads, "deconv3", "gA", self.shape(1, 32), "b2", "gB", self.shape(2, 64), True)

    def _group_deconv2(self, v, grads):
        self._deconv_group(v, grads, "deconv2", "gB", self.shape(2, 64), "b1", "gA", self.shape(3, 128), True)

    def _group_deconv1(self, v, grads):
        self._deconv_group(v, grads, "deconv1", "gA", self.shape(3, 128), "d1", "gB", self.shape(4, 256), False)

    def _group_dense1(self, v, grads):
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        feat = int(np.prod(self.s[4])) * 256
        gin = self._grad_view(v["g"]["gB"], (B, feat))
        j.finite("dense1 input gradient", gin)
        L.check_reduction(j, "dense1.wgrad", grads["decoder/dense1/kernel"],
                          lambda dt, f0, f1: op(v["z"], False, dt, f0, f1)[:, :z].T @ gin[f0:f1].to(dt), B, taps=False)
        L.check_reduction(j, "dense1.bias", grads["decoder/dense1/bias"], lambda dt, f0, f1: gin[f0:f1].to(dt).sum(0), B, taps=False)
        with self.feat_floor():
            L.check_frames(j, "dense1.dgrad", v["gz"][:, :z],
                           lambda dt, f0, f1: gin[f0:f1].to(dt) @ wt("decoder/dense1/kernel", False, dt).T, B)
        if not bool((v["gz"][:, z:] == 0).all()):
            j.failures.append("dense1.dgrad %s: padded columns of gz are not 0" % j.tag)

    def _group_heads(self, v, grads):
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        gh = v["gheads"]
        j.finite("heads input gradient", gh[:, :, :z])
        a4 = v["a4"].reshape(B, -1)
        for i, name in enumerate(("mean", "logstd_sqare")):
            L.check_reduction(j, "heads.wgrad (%s)" % name, grads[name + "/kernel"],
                              lambda dt, f0, f1, i=i: a4[f0:f1].to(dt).T @ gh[i, f0:f1, :z].to(dt), B, taps=False)
            L.check_reduction(j, "heads.bias (%s)" % name, grads[name + "/bias"],
                              lambda dt, f0, f1, i=i: gh[i, f0:f1, :z].to(dt).sum(0), B, taps=False)
        out = self._grad_view(v["g"]["gA"], self.shape(4, 256))
        L.check_frames(j, "heads.dgrad", out, lambda dt, f0, f1: (
            L.R.heads_dgrad(gh[:, f0:f1].to(dt), wt("mean/kernel", False, dt), wt("logstd_sqare/kernel", False, dt))
            .reshape((f1 - f0,) + self.s[4] + (256,)) * (v["a4"][f0:f1] > 0)), B)

    def _group_conv4(self, v, grads):
        self._enc_group(v, grads, "conv4", "gA", self.shape(4, 256), "a3", "gB", self.shape(3, 128))

    def _group_conv3(self, v, grads):
        self._enc_group(v, grads, "conv3", "gB", self.shape(3, 128), "a2", "gA", self.shape(2, 64))

    def _group_conv2(self, v, grads):
        op = self._op
        self._enc_group(v, grads, "conv2", "gA", self.shape(2, 64), "a1", "gB", self.shape(1, 32))
        gin = self._grad_view(v["g"]["gB"], self.shape(1, 32))
        self._conv_group(grads, "conv1", "encoder/conv1", gin,
                         lambda dt, f0, f1: (op(v["xp"], False, dt, f0, f1)[..., :3], op(gin, False, dt, f0, f1)))


LAYER_CASES = [(g, b, 3, 64) for g in GEOMETRIES if g != (512, 512) for b in (1, 3, 43, 257)] + \
              [(g, 3, 1, 100) for g in ((64, 96), (112, 208))] + [((160, 320), 1024, 3, 64), ((512, 512), 2, 3, 64)]


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["simt", "tc3xtf32", "tf32"])
@pytest.mark.parametrize("hw,batch,ct,z", LAYER_CASES, ids=["%dx%d-B%d-ct%d-z%d" % (c[0] + c[1:]) for c in LAYER_CASES])
def test_every_layer_pass_on_the_devices_own_operands(lib, tmp_path, hw, batch, ct, z, mode):
    allow = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        case = GeoCase(lib, tmp_path, mode, batch, ct, z, hw)
        case.forward()
        case.backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = allow
    assert not case.j.failures, "\n".join(case.j.failures[:40])


# --------------------------------------------------------------------------------------------------- 80x160 bit identity
def _legacy_vs_spec(lib, vae, batch, mode):
    """Every compute entry point through cpb_vae_* and cpb_vae_spec_* on the same inputs: outputs and launch counts."""
    from carla_ppo_b200 import _lib
    from carla_ppo_b200.ppo import PPO
    from helpers import Box
    _lib.check(lib.cpb_set_math_mode(mode))
    rs = np.random.RandomState(batch)
    x = torch.as_tensor(rs.randint(0, 256, size=(batch, 80, 160, 3)).astype(np.uint8), device=vae._device)
    xf = x.float() / 255
    eps = torch.as_tensor(rs.randn(batch, 64).astype(np.float32), device=vae._device)
    cfg_u8 = vae._base_config(batch, _lib.FRAME_U8, _lib.FRAME_U8)
    cfg = vae._base_config(batch)
    spec_u8, spec = vae._config(batch, _lib.FRAME_U8, _lib.FRAME_U8), vae._config(batch)
    ppo = PPO((67,), Box(np.array([-1., 0.]), np.array([1., 1.])), model_dir=os.path.join(vae.model_dir, "ppo"), seed=0)
    ppo.init_session(init_logging=False)
    p0 = vae.params.clone()
    P = _lib.ptr
    ws_tr, ws_enc = vae._workspace(batch, _lib.WS_TRAIN), vae._workspace(batch, _lib.WS_ENCODE)
    ws_p = ppo._workspace(batch)
    stream = vae._stream()
    meas = torch.as_tensor(rs.rand(batch, 3).astype(np.float32), device=vae._device)
    noise = torch.as_tensor(rs.randn(batch, 2).astype(np.float32), device=vae._device)

    def run(legacy):
        c, cu = (cfg, cfg_u8) if legacy else (spec, spec_u8)
        name = lambda n: "cpb_" + (n if legacy else n.replace("vae_", "vae_spec_"))
        out, counts = {}, {}
        vae.params.copy_(p0)
        vae.adam_m.zero_(); vae.adam_v.zero_(); vae.adam_powers.copy_(torch.tensor([0.9, 0.999]))

        def call(label, fn, *args):
            torch.cuda.synchronize()
            lib.cpb_reset_launch_count()
            _lib.check(getattr(lib, fn)(*args), fn)
            torch.cuda.synchronize()
            counts[label] = lib.cpb_launch_count()
        mean = torch.empty(batch, 64, device=vae._device)
        call("encode", name("vae_encode"), C.byref(cu), P(vae.params), P(x), P(mean), None, None, P(ws_tr), ws_tr.numel(), stream)
        out["encode"] = mean.clone()
        rec = torch.empty(batch, 80 * 160 * 3, device=vae._device)
        call("decode", name("vae_decode"), C.byref(c), P(vae.params), P(eps), P(rec), P(ws_tr), ws_tr.numel(), stream)
        out["decode"] = rec.clone()
        losses = torch.empty(2, device=vae._device)
        lat = [torch.empty(batch, 64, device=vae._device) for _ in range(3)]
        call("forward", name("vae_forward"), C.byref(c), P(vae.params), P(xf), P(xf), P(eps), P(losses), *[P(t) for t in lat],
             P(rec), None, P(ws_tr), ws_tr.numel(), stream)
        out["forward"] = torch.cat([losses] + [t.reshape(-1) for t in lat] + [rec.reshape(-1)])
        call("loss_grad", name("vae_loss_grad"), C.byref(c), P(vae.params), P(xf), P(xf), P(eps), P(vae.grads), P(losses), None,
             P(ws_tr), ws_tr.numel(), stream)
        out["loss_grad"] = torch.cat([vae.grads, losses])
        call("train_step", name("vae_train_step"), C.byref(c), P(vae.params), P(vae.grads), P(vae.adam_m), P(vae.adam_v),
             P(vae.adam_powers), 1e-4, P(xf), P(xf), P(eps), P(losses), None, P(ws_tr), ws_tr.numel(), stream)
        out["train_step"] = torch.cat([vae.params, vae.adam_m, vae.adam_v, losses])
        need = getattr(lib, name("vae_staging_bytes"))(C.byref(cu))
        st = torch.empty(int(need), dtype=torch.uint8, device=vae._device)
        xh, eh = x.cpu().numpy(), eps.cpu().numpy()
        lh = np.zeros(2, np.float32)
        call("train_step_host", name("vae_train_step_host"), C.byref(cu), P(vae.params), P(vae.grads), P(vae.adam_m),
             P(vae.adam_v), P(vae.adam_powers), 1e-4, P(xh), P(xh), P(eh), P(lh), None, P(st), st.numel(), P(ws_tr),
             ws_tr.numel(), stream)
        out["train_step_host"] = torch.cat([vae.params, vae.adam_m, vae.adam_v, torch.as_tensor(lh, device=vae._device)])
        state = torch.empty(batch, 67, device=vae._device)
        act, val = torch.empty(batch, 2, device=vae._device), torch.empty(batch, device=vae._device)
        fn = "cpb_encode_predict" if legacy else "cpb_vae_spec_encode_predict"
        call("encode_predict", fn, C.byref(cu), P(vae.params), P(x), P(meas), 3, C.byref(ppo._c), P(ppo.params), P(noise),
             P(mean), P(state), P(act), P(val), None, P(ws_enc), ws_enc.numel(), P(ws_p), ws_p.numel(), stream)
        out["encode_predict"] = torch.cat([state.reshape(-1), act.reshape(-1), val])
        return out, counts
    return run(True), run(False)


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["simt", "tc3xtf32", "tf32"])
@pytest.mark.parametrize("batch", [1, 33])
def test_legacy_and_spec_entry_points_are_bit_identical_at_80x160(lib, tmp_path, mode, batch):
    from helpers import shipped_vae_weights
    vae = make_vae(tmp_path, (80, 160), 3, "bce", 64, shipped_vae_weights()[0])
    (lo, lc), (so, sc) = _legacy_vs_spec(lib, vae, batch, mode)
    assert lc == sc
    for k in lo:
        assert torch.equal(lo[k], so[k]), k
        assert bool(torch.isfinite(lo[k]).all()), k


# --------------------------------------------------------------------------------------------------- batch bound
def tc_bound(h, w):
    return ((1 << 31) - 1) // ((h // 2 - 1) * (w // 2 - 1) * 32)


@pytest.mark.parametrize("mode", [1, 2])
def test_batch_bound(lib, tmp_path, mode):
    """B = bound + 1 is refused with CPB_ERR_UNSUPPORTED and no launch; at 512x512 the bound itself (1032 frames) runs,
    and its first frames encode as they do in a batch of 2."""
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_set_math_mode(mode))
    for hw in ((80, 160), (160, 320), (512, 512)):
        vae = make_vae(tmp_path, hw, tag="b%d" % hw[0])
        bound = tc_bound(*hw)
        spec = vae._config(bound + 1, _lib.FRAME_U8)
        ws = vae._workspace(2, _lib.WS_ENCODE)
        lib.cpb_reset_launch_count()
        mean = torch.empty(2, 64, device=vae._device)
        rc = lib.cpb_vae_spec_encode(C.byref(spec), _lib.ptr(vae.params), _lib.ptr(ws), _lib.ptr(mean), None, None,
                                     _lib.ptr(ws), 1 << 40, vae._stream())
        assert rc == -4 and b"above %d" % bound in lib.cpb_last_error()
        assert lib.cpb_launch_count() == 0
    # 512x512 at the bound: ~20 GB of encode workspace
    torch.cuda.empty_cache()
    vae = make_vae(tmp_path, (512, 512), tag="run")
    bound = tc_bound(512, 512)
    frames = torch.randint(0, 256, (bound, 512, 512, 3), dtype=torch.uint8, device=vae._device)
    mean = vae.encode_device(frames)
    torch.cuda.synchronize()
    small = vae.encode_device(frames[:2].contiguous())
    assert bool(torch.isfinite(mean).all())
    assert rel_l2(mean[:2].cpu().numpy(), small.cpu().numpy()) < 1e-5
    vae._ws.clear()
    del frames
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------------- RL path at 64x128
def frames_64x128(n=48):
    rgb, _ = committed_frames()
    return np.ascontiguousarray(np.stack([rgb[i % len(rgb)][8:72, 16:144] for i in range(n)]))


@pytest.mark.parametrize("n", [1, 4])
def test_fused_actor_at_64x128(lib, tmp_path, n):
    from carla_ppo_b200.actor import FusedActor, UnfusedActor
    from carla_ppo_b200.ppo import PPO
    from helpers import Box
    vae = make_vae(tmp_path, (64, 128), training=False)
    frames = frames_64x128()
    envs = []
    for i in range(n):
        v = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.1 * i - 0.2, throttle=0.3), get_speed=(lambda s=0.5 * i: s))
        envs.append(types.SimpleNamespace(observation=frames[3 * i], vehicle=v))
    models = []
    for tag in ("fused", "unfused"):
        m = PPO((67,), Box(np.array([-1., 0.]), np.array([1., 1.])), initial_std=0.4, model_dir=str(tmp_path / tag), seed=0)
        m.init_session(init_logging=False)
        models.append(m)
    meas = ("steer", "throttle", "speed")
    fs, fa, fv = FusedActor(vae, models[0], meas).encode_predict(envs)
    us, ua, uv = UnfusedActor(vae, models[1], meas).encode_predict(envs)
    assert all(np.array_equal(a, b) for a, b in zip(fs, us))
    assert np.array_equal(fa, ua) and np.array_equal(fv, uv)


def test_train_from_a_64x128_checkpoint(lib, tmp_path):
    """ConvVAE.save records the frame size; load_vae rebuilds the model from it; train.train builds its replay
    environments at that size and runs the fused actor for one round."""
    from carla_ppo_b200.train import train
    from carla_ppo_b200.vae_common import load_vae
    from test_integration_gpu import _train_params
    model_dir = str(tmp_path / "rgb_mse_cnn_zdim64")
    vae = make_vae(tmp_path, (64, 128), tag="rgb_mse_cnn_zdim64")
    x = frames_64x128(8)
    vae.train_step(x, x)
    vae.save()
    loaded = load_vae(model_dir)
    assert loaded.source_shape == (64, 128, 3) and loaded.encoded_shape == (2, 6, 256)
    assert all(np.array_equal(a, loaded.get_weights()[k]) for k, a in vae.get_weights().items())
    assert load_vae(model_dir, source_shape=(64, 128, 3)).source_shape == (64, 128, 3)
    # an explicit shape that disagrees with the checkpoint's is refused (the layouts of 64x128 and 128x64 coincide)
    with pytest.raises(Exception, match="Failed to load VAE"):
        load_vae(model_dir, source_shape=(128, 64, 3))
    data = str(tmp_path / "replay.npz")
    np.savez(data, rgb=frames_64x128(40))
    params = _train_params("fs", num_episodes=1, replay_data=data, episode_length=24)
    model = train(params, restart=False, vae=loaded, models_root=str(tmp_path / "models"), interactive=False)
    assert model.get_episode_idx() == 1


def test_train_vae_cli_on_64x128_pngs(lib, tmp_path):
    from PIL import Image
    from carla_ppo_b200.vae import train_vae
    from carla_ppo_b200.vae_common import load_vae
    d = tmp_path / "data" / "rgb"
    d.mkdir(parents=True)
    for i, f in enumerate(frames_64x128(40)):
        Image.fromarray(f).save(str(d / ("%d.png" % i)))
    vae = train_vae.main(["--dataset", str(tmp_path / "data"), "--model_name", "rgb_bce_cnn_zdim64_fs", "--batch_size", "8",
                          "--max_epochs", "2", "--models_root", str(tmp_path / "models")])
    assert vae.source_shape == (64, 128, 3) and vae.get_step_idx() == 2
    loaded = load_vae(str(tmp_path / "models" / "rgb_bce_cnn_zdim64_fs"))
    assert loaded.source_shape == (64, 128, 3)
