"""Every ConvVAE layer pass on the operands the device itself computed, judged against float64 (tests/vae_layer_ref.py):
the checks of tests/test_vae_layers_gpu.py, tests/test_frame_size_gpu.py and tests/test_large_batch_gpu.py.

Gate: max(FLOOR, 2 x err_f32), err_f32 = the distance from float64 of the same formulation evaluated in float32 with
TF32 off on the same slice (the caller turns it off)."""
import numpy as np
import torch

import vae_layer_ref as R
from harness import conv_workspace, make_conv_vae, sides

FLOOR = 2e-6
CHUNK = 256          # frames per reference evaluation (the float64 im2col of deconv3's data gradient: 1.1 GB)
ZCHUNK = 1 << 26     # elements per step of Judge.zeros

STOPS = ["deconv4.dgrad", "deconv3.dgrad", "deconv2.dgrad", "deconv1.dgrad", "dense1.dgrad", "heads.dgrad",
         "conv4.dgrad", "conv3.dgrad", None]
# the parameter tensors whose gradients each layer group writes, in pass order (None: the rest of the pass)
GROUP_TENSORS = [["decoder/deconv4"], ["decoder/deconv3"], ["decoder/deconv2"], ["decoder/deconv1"], ["decoder/dense1"],
                 ["mean", "logstd_sqare"], ["encoder/conv4"], ["encoder/conv3"], ["encoder/conv2", "encoder/conv1"]]


class Judge:
    """Collects, per named slice, ||dev - ref64||^2, ||ref32 - ref64||^2 and ||ref64||^2, and gates each slice at
    max(floor, 2 x its own err_f32).  Failures are collected so that one run names every broken pass."""

    def __init__(self, tag):
        self.tag = tag
        self.failures = []
        self.worst = {}
        self.live = None

    def zeros(self, what, t):
        """Placed-frame batches (self.live: the sorted live frames): every null frame of t [B, ...] exactly 0 (a NaN
        left by a missed write is not 0), every live frame finite.  Reduced per frame, in chunks, on the device."""
        live = torch.zeros(t.shape[0], dtype=torch.bool, device=t.device)
        live[self.live] = True
        step = max(1, ZCHUNK // max(1, t[0].numel()))
        for f0 in range(0, t.shape[0], step):
            c = t[f0:f0 + step].reshape(min(step, t.shape[0] - f0), -1)
            bad = torch.where(live[f0:f0 + step], ~torch.isfinite(c).all(1), (c != 0).any(1))
            if bool(bad.any()):
                frames = (torch.nonzero(bad)[:, 0] + f0).tolist()
                self.failures.append("%s %s: frames %s%s are %s" % (what, self.tag, frames[:8], " ..." if len(frames) > 8 else "",
                                     "not finite (live)" if frames[0] in self.live else "not 0 (null frame)"))
                return

    def finite(self, what, t):
        if not bool(torch.isfinite(t).all()):
            bad = torch.nonzero(~torch.isfinite(t))[0].tolist()
            self.failures.append("%s %s: non-finite output at %s" % (what, self.tag, bad))

    def gate(self, what, slice_name, dd, ff, rr, floor=FLOOR):
        """dd, ff, rr: float64 tensors of per-slice sums of squares (same shape)."""
        dd, ff, rr = dd.double(), ff.double(), rr.double()
        pos = rr > 0
        err = torch.where(pos, torch.sqrt(dd / torch.where(pos, rr, torch.ones_like(rr))),
                          torch.where(dd > 0, torch.full_like(dd, float("inf")), torch.zeros_like(dd)))
        e32 = torch.where(pos, torch.sqrt(ff / torch.where(pos, rr, torch.ones_like(rr))), torch.zeros_like(ff))
        gate = torch.clamp(2.0 * e32, min=floor)
        ratio = err / gate
        worst = int(torch.argmax(ratio.reshape(-1)))
        r = float(ratio.reshape(-1)[worst])
        self.worst[what] = max(self.worst.get(what, 0.0), r)
        if not r <= 1.0:
            idx = [int(i) for i in np.unravel_index(worst, tuple(ratio.shape))] if ratio.dim() else []
            self.failures.append("%s %s: %s%s rel err %.3e > gate %.3e (err_f32 %.3e)" % (
                what, self.tag, slice_name, " %s" % idx if idx else "", float(err.reshape(-1)[worst]),
                float(gate.reshape(-1)[worst]), float(e32.reshape(-1)[worst])))

    def report(self):
        print("\n%s: worst err/gate %s" % (self.tag, ", ".join("%s %.2f" % kv for kv in sorted(self.worst.items(), key=lambda kv: -kv[1])[:6])))
        assert not self.failures, "\n".join(self.failures[:40])


def _sq(a, b, dims):
    d = a.double() - b
    return (d * d).sum(dims)


def spans(frames):
    """The frame ranges (f0, f1) a check visits: chunks of CHUNK frames over a whole batch of `frames`, or the given list
    of ranges (the live frames of a placed-frame batch)."""
    if isinstance(frames, int):
        return [(f0, min(frames, f0 + CHUNK)) for f0 in range(0, frames, CHUNK)]
    return frames


def check_frames(j, what, dev, ref, B, floor=FLOOR):
    """dev: the device's [B, ...] output; ref(dtype, f0, f1): the reference for frames f0:f1.  Gates the whole tensor,
    every frame and, for images, the first / last row and column of every frame, over the frames spans(B) names; in a
    placed-frame batch (j.live) every other frame must be exactly 0."""
    image = dev.dim() == 4
    names = ["frame"] + (["first row", "last row", "first column", "last column"] if image else [])
    sums = {n: [[], [], []] for n in names}
    if j.live is not None:
        j.zeros(what, dev)
    for f0, f1 in spans(B):
        d = dev[f0:f1]
        j.finite(what, d)
        r64 = ref(torch.float64, f0, f1)
        r32 = ref(torch.float32, f0, f1)
        parts = {"frame": (d, r64, r32)}
        if image:
            parts.update({"first row": (d[:, 0], r64[:, 0], r32[:, 0]), "last row": (d[:, -1], r64[:, -1], r32[:, -1]),
                          "first column": (d[:, :, 0], r64[:, :, 0], r32[:, :, 0]),
                          "last column": (d[:, :, -1], r64[:, :, -1], r32[:, :, -1])})
        for n, (a, b64, b32) in parts.items():
            dims = tuple(range(1, a.dim()))
            sums[n][0].append(_sq(a, b64, dims))
            sums[n][1].append(_sq(b32, b64, dims))
            sums[n][2].append((b64 * b64).sum(dims))
        del r64, r32
    dd, ff, rr = (torch.cat(s) for s in sums["frame"])
    j.gate(what, "whole tensor", dd.sum(), ff.sum(), rr.sum(), floor)
    for n in names:
        j.gate(what, n if n == "frame" else n + " of frame", *(torch.cat(s) for s in sums[n]), floor)


def check_reduction(j, what, dev, ref, B, taps):
    """dev: the device's weight or bias gradient; ref(dtype, f0, f1): the contribution of frames f0:f1 (summed over
    spans(B) in that dtype: in a placed-frame batch, whose null frames contribute exactly 0, the live frames alone).  Gates the whole tensor and, for a conv kernel [k, k, Cb, Cs], every tap block."""
    j.finite(what, dev)
    r64 = r32 = 0
    for f0, f1 in spans(B):
        r64 = r64 + ref(torch.float64, f0, f1)
        r32 = r32 + ref(torch.float32, f0, f1)
    dims = tuple(range(dev.dim()))
    j.gate(what, "whole tensor", _sq(dev, r64, dims), _sq(r32, r64, dims), (r64 * r64).sum())
    if taps:
        j.gate(what, "tap block (kh, kw) =", _sq(dev, r64, (2, 3)), _sq(r32, r64, (2, 3)), (r64 * r64).sum((2, 3)))


class Case:
    """One model, batch and math mode (the caller sets the mode).  forward() and backward() check every layer pass of
    a forward and of a training call.  hw: the frame size, 80x160 when None (the two are seeded differently)."""
    dgrad = True         # False: backward() checks the weight and bias gradients only (the reductions over the batch)

    def __init__(self, lib, tmp_path, mode, B, ct, z, hw=None):
        from oracle import vae_oracle as vo
        h, w = hw or (80, 160)
        seed_h, seed_w = (0, 0) if hw is None else hw
        self.s = sides(h, w)
        self.lib, self.mode, self.B, self.ct, self.z = lib, mode, B, ct, z
        self.frames = B      # what the checks visit (spans): the whole batch, or the live frames of a placed-frame batch
        self.j = Judge(("%dx%d " % hw if hw else "") + "mode %d B=%d ct=%d z=%d" % (mode, B, ct, z))
        wts = vo.glorot_init(B + 10 * ct + seed_h, (h, w, 3), ct, z)
        rs = np.random.RandomState(B + ct + seed_w)
        for k in wts:
            if k.endswith("bias"):       # biases that move the ReLU kinks and that the bias gradient paths must add
                wts[k] = (0.05 * rs.randn(*wts[k].shape)).astype(np.float32)
        self.vae = make_conv_vae(tmp_path, wts, (h, w), ct, "mse" if ct == 3 else "bce", z)
        d = self.vae._device
        self.w = {k: torch.from_numpy(v).to(d) for k, v in wts.items()}
        g = torch.Generator(device=d)
        g.manual_seed(1000 + B)
        self.x = torch.rand(B, h, w, 3, generator=g, device=d)
        self.y = self.x if ct == 3 else torch.rand(B, h, w, 1, generator=g, device=d)
        self.eps = torch.randn(B, z, generator=g, device=d)

    def shape(self, level, c):
        return (self.B,) + self.s[level] + (c,)

    def feat_floor(self):
        """The gate floor of a reduction over the FEAT = H4*W4*256 features (heads forward, dense1's data gradient):
        FLOOR holds for FEAT = 6144 (80x160); the rounding error of a serial fp32 sum grows as the square root of its
        length, so the floor scales by sqrt(FEAT / 6144) above it (x 6.1 at 512x512)."""
        return FLOOR * max(1.0, np.sqrt(int(np.prod(self.s[4])) * 256 / 6144))

    # -------------------------------------------------------------- workspace
    def _poisoned(self, ws_mode):
        ws = self.vae._workspace(self.B, ws_mode)
        ws.fill_(0xFF)
        return ws

    def _views(self, ws_mode):
        return conv_workspace(self.vae, self.B, ws_mode)

    @staticmethod
    def _grad_view(raw, shape):
        """The first prod(shape) floats of a ping-pong gradient buffer (sized for the largest layer) as `shape`."""
        return raw[:4 * int(np.prod(shape))].view(torch.float32).view(shape)

    # -------------------------------------------------------------- reference helpers
    def _op(self, t, tc, dtype, f0=None, f1=None):
        """An operand of a contraction: frames f0:f1 of t (all of t for a weight), rounded to TF32 first when the
        contraction runs on the tensor cores in mode 2."""
        if f0 is not None:
            t = t[f0:f1]
        if tc and self.mode == 2:
            t = R.round_tf32(t)
        return t.to(dtype)

    def _wt(self, name, tc, dtype):
        return self._op(self.w[name], tc, dtype)

    # -------------------------------------------------------------- forward
    def forward(self, encode_only=False):
        """encode_only: an encode call, its encoder passes and heads checked in the encode workspace."""
        from carla_ppo_b200 import _lib
        ws_mode = _lib.WS_ENCODE if encode_only else _lib.WS_FORWARD
        self._poisoned(ws_mode)
        if encode_only:
            self.vae.encode_device(self.x)
        else:
            self.losses = self.vae.forward_device(self.x, self.y, self.eps)["losses"]
        torch.cuda.synchronize()
        v = self._views(ws_mode)
        j, z, op, wt, s = self.j, self.z, self._op, self._wt, self.s
        relu = torch.relu

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

        check_frames(j, "conv1.fwd", v["a1"], conv("conv1", "xp", False), self.frames)
        check_frames(j, "conv2.fwd", v["a2"], conv("conv2", "a1", True), self.frames)
        check_frames(j, "conv3.fwd", v["a3"], conv("conv3", "a2", True), self.frames)
        check_frames(j, "conv4.fwd", v["a4"], conv("conv4", "a3", True), self.frames)
        for i, name in enumerate(("mean", "logstd_sqare")):
            check_frames(j, "heads.fwd (%s)" % name, v["heads"][i, :, :z], lambda dt, f0, f1, name=name: (
                op(v["a4"], False, dt, f0, f1).reshape(f1 - f0, -1) @ wt(name + "/kernel", False, dt)
                + self.w[name + "/bias"].to(dt)), self.frames, self.feat_floor())
        if not bool((v["heads"][:, :, z:] == 0).all()):
            j.failures.append("heads.fwd %s: padded columns are not 0" % j.tag)
        if encode_only:
            return
        check_frames(j, "dense1.fwd", v["d1"], lambda dt, f0, f1: (
            R.dense1_fwd(op(v["z"], False, dt, f0, f1), wt("decoder/dense1/kernel", False, dt))
            + self.w["decoder/dense1/bias"].to(dt)).reshape((f1 - f0,) + s[4] + (256,)), self.frames)
        check_frames(j, "deconv1.fwd", v["b1"], deconv("deconv1", "d1", True, s[3]), self.frames)
        check_frames(j, "deconv2.fwd", v["b2"], deconv("deconv2", "b1", True, s[2]), self.frames)
        check_frames(j, "deconv3.fwd", v["b3"], deconv("deconv3", "b2", True, s[1]), self.frames)
        check_frames(j, "deconv4.fwd", v["logits_p"][..., :self.ct], deconv("deconv4", "b3", False, s[0], act=False), self.frames)

    # -------------------------------------------------------------- backward
    def backward(self):
        from carla_ppo_b200 import _lib
        for gi, stop in enumerate(STOPS):
            _lib.check(self.lib.cpb_debug_vae_backward_stop(stop.encode() if stop else None))
            self._poisoned(_lib.WS_TRAIN)
            self.vae.grads.fill_(float("nan"))
            self.vae.loss_grad_device(self.x, self.y, self.eps)
            torch.cuda.synchronize()
            v = self._views(_lib.WS_TRAIN)
            grads = {k: torch.from_numpy(a).to(self.vae._device) for k, a in self.vae.get_grads().items()}
            for later in GROUP_TENSORS[gi + 1:]:
                for t in later:
                    for suffix in ("/kernel", "/bias"):
                        if not bool((grads[t + suffix] == 0).all()):
                            self.j.failures.append("stop %s %s: %s%s is not 0" % (stop, self.j.tag, t, suffix))
            getattr(self, "_group_" + (stop or "conv2.dgrad").split(".")[0])(v, grads)

    def _conv_group(self, grads, name, prefix, gin, wgrad_ops, dgrad=None):
        """One layer group: weight gradient from wgrad_ops(dt, f0, f1) -> (big, small), bias gradient = the sum of the
        input gradient gin, and (if given) the data gradient dgrad = (device output, ref)."""
        j, k = self.j, self.w[prefix + "/kernel"].shape[0]
        check_reduction(j, name + ".wgrad", grads[prefix + "/kernel"],
                        lambda dt, f0, f1: R.wgrad(*wgrad_ops(dt, f0, f1), k), self.frames, taps=True)
        check_reduction(j, name + ".bias", grads[prefix + "/bias"],
                        lambda dt, f0, f1: gin[f0:f1].to(dt).sum((0, 1, 2)), self.frames, taps=False)
        if dgrad is not None and self.dgrad:
            check_frames(j, name + ".dgrad", dgrad[0], dgrad[1], self.frames)

    def _group_deconv4(self, v, grads):
        ct, op, wt = self.ct, self._op, self._wt
        dlog = v["logits_p"][..., :ct]
        gA = self._grad_view(v["g"]["gA"], self.shape(1, 32))
        self.j.finite("deconv4 input gradient", dlog)
        self._conv_group(grads, "deconv4", "decoder/deconv4", dlog,
                         lambda dt, f0, f1: (op(dlog, False, dt, f0, f1), op(v["b3"], False, dt, f0, f1)),
                         (gA, lambda dt, f0, f1: R.gather(op(dlog, False, dt, f0, f1), wt("decoder/deconv4/kernel", False, dt))
                          * (v["b3"][f0:f1] > 0)))

    def _deconv_group(self, v, grads, name, gin_name, gin_shape, below, out_name, out_shape, masked):
        op, wt = self._op, self._wt
        gin = self._grad_view(v["g"][gin_name], gin_shape)
        out = self._grad_view(v["g"][out_name], out_shape)
        self.j.finite(name + " input gradient", gin)

        def dref(dt, f0, f1):
            r = R.gather(op(gin, True, dt, f0, f1), wt("decoder/%s/kernel" % name, True, dt))
            return r * (v[below][f0:f1] > 0) if masked else r
        self._conv_group(grads, name, "decoder/" + name, gin,
                         lambda dt, f0, f1: (op(gin, True, dt, f0, f1), op(v[below], True, dt, f0, f1)), (out, dref))

    def _group_deconv3(self, v, grads):
        self._deconv_group(v, grads, "deconv3", "gA", self.shape(1, 32), "b2", "gB", self.shape(2, 64), True)

    def _group_deconv2(self, v, grads):
        self._deconv_group(v, grads, "deconv2", "gB", self.shape(2, 64), "b1", "gA", self.shape(3, 128), True)

    def _group_deconv1(self, v, grads):
        self._deconv_group(v, grads, "deconv1", "gA", self.shape(3, 128), "d1", "gB", self.shape(4, 256), False)

    def _group_dense1(self, v, grads):
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        gin = self._grad_view(v["g"]["gB"], (B, int(np.prod(self.s[4])) * 256))
        j.finite("dense1 input gradient", gin)
        check_reduction(j, "dense1.wgrad", grads["decoder/dense1/kernel"],
                        lambda dt, f0, f1: op(v["z"], False, dt, f0, f1)[:, :z].T @ gin[f0:f1].to(dt), self.frames, taps=False)
        check_reduction(j, "dense1.bias", grads["decoder/dense1/bias"], lambda dt, f0, f1: gin[f0:f1].to(dt).sum(0), self.frames, taps=False)
        if self.dgrad:
            check_frames(j, "dense1.dgrad", v["gz"][:, :z],
                         lambda dt, f0, f1: gin[f0:f1].to(dt) @ wt("decoder/dense1/kernel", False, dt).T, self.frames,
                         self.feat_floor())
        if not bool((v["gz"][:, z:] == 0).all()):
            j.failures.append("dense1.dgrad %s: padded columns of gz are not 0" % j.tag)

    def _group_heads(self, v, grads):
        j, B, z, wt = self.j, self.B, self.z, self._wt
        gh = v["gheads"]
        j.finite("heads input gradient", gh[:, :, :z])
        a4 = v["a4"].reshape(B, -1)
        for i, name in enumerate(("mean", "logstd_sqare")):
            check_reduction(j, "heads.wgrad (%s)" % name, grads[name + "/kernel"],
                            lambda dt, f0, f1, i=i: a4[f0:f1].to(dt).T @ gh[i, f0:f1, :z].to(dt), self.frames, taps=False)
            check_reduction(j, "heads.bias (%s)" % name, grads[name + "/bias"],
                            lambda dt, f0, f1, i=i: gh[i, f0:f1, :z].to(dt).sum(0), self.frames, taps=False)
        out = self._grad_view(v["g"]["gA"], self.shape(4, 256))
        if self.dgrad:
            check_frames(j, "heads.dgrad", out, lambda dt, f0, f1: (
                R.heads_dgrad(gh[:, f0:f1].to(dt), wt("mean/kernel", False, dt), wt("logstd_sqare/kernel", False, dt))
                .reshape((f1 - f0,) + self.s[4] + (256,)) * (v["a4"][f0:f1] > 0)), self.frames)

    def _enc_group(self, v, grads, name, gin_name, gin_shape, src, out_name, out_shape):
        op, wt = self._op, self._wt
        gin = self._grad_view(v["g"][gin_name], gin_shape)
        out = self._grad_view(v["g"][out_name], out_shape)
        self.j.finite(name + " input gradient", gin)
        self._conv_group(grads, name, "encoder/" + name, gin,
                         lambda dt, f0, f1: (op(v[src], True, dt, f0, f1), op(gin, True, dt, f0, f1)),
                         (out, lambda dt, f0, f1: R.scatter(op(gin, True, dt, f0, f1), wt("encoder/%s/kernel" % name, True, dt),
                                                            out_shape[1:3]) * (v[src][f0:f1] > 0)))

    def _group_conv4(self, v, grads):
        self._enc_group(v, grads, "conv4", "gA", self.shape(4, 256), "a3", "gB", self.shape(3, 128))

    def _group_conv3(self, v, grads):
        self._enc_group(v, grads, "conv3", "gB", self.shape(3, 128), "a2", "gA", self.shape(2, 64))

    def _group_conv2(self, v, grads):
        # the whole pass: conv2's group, then conv1's weight and bias gradient from conv2's output gradient
        op = self._op
        self._enc_group(v, grads, "conv2", "gA", self.shape(2, 64), "a1", "gB", self.shape(1, 32))
        gin = self._grad_view(v["g"]["gB"], self.shape(1, 32))
        self._conv_group(grads, "conv1", "encoder/conv1", gin,
                         lambda dt, f0, f1: (op(v["xp"], False, dt, f0, f1)[..., :3], op(gin, False, dt, f0, f1)))
