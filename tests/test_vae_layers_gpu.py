"""Every ConvVAE layer pass on the operands the device itself computed, in math modes 0, 1 and 2, from one frame to the
shipping batch.

Each pass -- forward, data gradient, weight gradient and bias gradient of every layer -- is read back from the
workspace (forward: the forward workspace, where logits_p holds the logits; backward: the training workspace, the
pass stopped with cpb_debug_vae_backward_stop right after the layer group under test, so that the ping-pong buffer the
group read still holds its input gradient) and compared with the same contraction in float64 on those operands
(tests/vae_layer_ref.py, pinned to the oracle by tests/test_vae_layers_cpu.py).  ReLU masks are the device's own
activations.  In math mode 2 both operands of exactly the 18 tensor-core contractions (forward, data and weight
gradient of conv2-4 and deconv1-3) are rounded with round_tf32 first.

Gate: max(2e-6, 2 x err_f32), err_f32 = the distance from float64 of the same formulation evaluated in float32 with
TF32 off on the same slice.  It is applied to the whole tensor, to every frame of a forward or data gradient, to the
first and last output row and column of every frame, and to every (kh, kw) tap block of a weight gradient.  The
workspace is filled with 0xFF bytes (NaN) before every call and every checked output must be finite; at each stop the
gradients of the layers the pass has not reached must be exactly 0.  A failure names the layer, pass, mode and batch."""
import ctypes as C

import numpy as np
import pytest
import torch

import vae_layer_ref as R

pytestmark = pytest.mark.gpu

FLOOR = 2e-6
CHUNK = 256          # frames per reference evaluation (the float64 im2col of deconv3's data gradient: 1.1 GB)
ZCHUNK = 1 << 26     # elements per step of Judge.zeros

# Batches and the edge each hits (M = B x positions per frame; tile and split rules in tapgemm.cu, tc_tapgemm.cu,
# wgrad.cu, tc_wgrad.cu):
#   1     every M below one 128-row tile; every weight gradient has one split (max_splits = ceil(M / 1024) = 1);
#   2     conv2 / deconv3 weight gradient (684 positions per frame): 2 splits of 704 positions, the boundary inside
#         frame 1 and the last split short (664);
#   3     deconv2 forward and conv3 data gradient (171 quads / class-(0,0) rows per frame): M = 513 = 4 x 128 + 1, so
#         the last 128-row tap-GEMM tile (tensor core, and the 64 / 128 / 256-row SIMT tiles) holds one valid row;
#   7     conv2 / deconv3 weight gradient: 5 splits of 960 positions, boundaries inside frames 1-5, the last split short;
#   33    conv3 / deconv2 weight gradient (144 positions per frame): 5 splits of 960 inside frames; one k-block of conv4
#         / deconv1 (24 positions per frame < 32) spans two frames, and 33 x 24 = 792 is not a multiple of 32;
#   43    conv4 / deconv1 weight gradient: M = 1032 > 1024, the first batch with 2 splits: 544 positions (inside frame
#         22) and a short last split of 488; the SIMT dense weight gradients (M = B) run 1 split;
#   257   the SIMT weight gradients of the heads and dense1: M = 257 > 256 gives 2 splits where 256 gives 1;
#   512   the 512-frame shard of a 4-GPU step;
#   4096  the one-GPU shipping batch: every weight gradient at its wave-filling split count, every frame gated.
# The k-split of the heads and of dense1's data gradient is a function of K = 6144 alone (tapgemm_pick_ksplit), so
# no batch changes it; z = 100 (z_pad = 128) changes their N and makes the library drop padded rows and columns.
CASES = [(b, 3, 64) for b in (1, 2, 3, 7, 33, 43, 257, 512, 4096)] + [(b, 1, 100) for b in (1, 3, 43, 512)]
MODES = [0, 1, 2]

BUFFERS = ["xp", "a1", "a2", "a3", "a4", "heads", "z", "d1", "b1", "b2", "b3", "logits_p", "gA", "gB", "frame_loss",
           "kl_rows", "gz", "gheads"]
STOPS = ["deconv4.dgrad", "deconv3.dgrad", "deconv2.dgrad", "deconv1.dgrad", "dense1.dgrad", "heads.dgrad",
         "conv4.dgrad", "conv3.dgrad", None]
# the parameter tensors whose gradients each layer group writes, in pass order (None: the rest of the pass)
GROUP_TENSORS = [["decoder/deconv4"], ["decoder/deconv3"], ["decoder/deconv2"], ["decoder/deconv1"], ["decoder/dense1"],
                 ["mean", "logstd_sqare"], ["encoder/conv4"], ["encoder/conv3"], ["encoder/conv2", "encoder/conv1"]]


@pytest.fixture(scope="module")
def lib():
    import os
    from carla_ppo_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(autouse=True)
def restore(lib):
    allow = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False      # err_f32: plain SGEMM
    yield
    torch.backends.cuda.matmul.allow_tf32 = allow
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_debug_vae_backward_stop(None))
    _lib.check(lib.cpb_set_math_mode(_lib.MATH_3XTF32))


class Judge:
    """Collects, per named slice, ||dev - ref64||^2, ||ref32 - ref64||^2 and ||ref64||^2, and gates each slice at
    max(FLOOR, 2 x its own err_f32).  Failures are collected so that one run names every broken pass."""

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

    def gate(self, what, slice_name, dd, ff, rr):
        """dd, ff, rr: float64 tensors of per-slice sums of squares (same shape)."""
        dd, ff, rr = dd.double(), ff.double(), rr.double()
        pos = rr > 0
        err = torch.where(pos, torch.sqrt(dd / torch.where(pos, rr, torch.ones_like(rr))),
                          torch.where(dd > 0, torch.full_like(dd, float("inf")), torch.zeros_like(dd)))
        e32 = torch.where(pos, torch.sqrt(ff / torch.where(pos, rr, torch.ones_like(rr))), torch.zeros_like(ff))
        gate = torch.clamp(2.0 * e32, min=FLOOR)
        ratio = err / gate
        worst = int(torch.argmax(ratio.reshape(-1)))
        r = float(ratio.reshape(-1)[worst])
        self.worst[what] = max(self.worst.get(what, 0.0), r)
        if not r <= 1.0:
            idx = [int(i) for i in np.unravel_index(worst, tuple(ratio.shape))] if ratio.dim() else []
            self.failures.append("%s %s: %s%s rel err %.3e > gate %.3e (err_f32 %.3e)" % (
                what, self.tag, slice_name, " %s" % idx if idx else "", float(err.reshape(-1)[worst]),
                float(gate.reshape(-1)[worst]), float(e32.reshape(-1)[worst])))


def _sq(a, b, dims):
    d = a.double() - b
    return (d * d).sum(dims)


def spans(frames):
    """The frame ranges (f0, f1) a check visits: chunks of CHUNK frames over a whole batch of `frames`, or the given list
    of ranges (the live frames of a placed-frame batch)."""
    if isinstance(frames, int):
        return [(f0, min(frames, f0 + CHUNK)) for f0 in range(0, frames, CHUNK)]
    return frames


def check_frames(j, what, dev, ref, B):
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
    j.gate(what, "whole tensor", dd.sum(), ff.sum(), rr.sum())
    for n in names:
        j.gate(what, n if n == "frame" else n + " of frame", *(torch.cat(s) for s in sums[n]))


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
    dgrad = True         # False: backward() checks the weight and bias gradients only (the reductions over the batch)

    def __init__(self, lib, tmp_path, mode, B, ct, z):
        from carla_ppo_b200 import _lib
        from carla_ppo_b200.vae.models import ConvVAE
        from oracle import vae_oracle as vo
        self.lib, self.mode, self.B, self.ct, self.z, self.zp = lib, mode, B, ct, z, 64 * ((z + 63) // 64)
        self.frames = B      # what the checks visit (spans): the whole batch, or the live frames of a placed-frame batch
        self.j = Judge("mode %d B=%d ct=%d z=%d" % (mode, B, ct, z))
        _lib.check(lib.cpb_set_math_mode(mode))
        w = vo.glorot_init(B + 10 * ct, target_channels=ct, z_dim=z)
        rs = np.random.RandomState(B + ct)
        for k in w:
            if k.endswith("bias"):       # biases that move the ReLU kinks and that the bias gradient paths must add
                w[k] = (0.05 * rs.randn(*w[k].shape)).astype(np.float32)
        self.vae = ConvVAE((80, 160, 3), target_shape=(80, 160, ct), z_dim=z, loss_fn="mse" if ct == 3 else "bce",
                           model_dir=str(tmp_path / "m"), seed=0)
        self.vae.init_session(init_logging=False)
        self.vae.set_weights(w)
        dev = self.vae._device
        self.w = {k: torch.from_numpy(v).to(dev) for k, v in w.items()}
        g = torch.Generator(device=dev)
        g.manual_seed(1000 + B)
        self.x = torch.rand(B, 80, 160, 3, generator=g, device=dev)
        self.y = self.x if ct == 3 else torch.rand(B, 80, 160, 1, generator=g, device=dev)
        self.eps = torch.randn(B, z, generator=g, device=dev)

    # -------------------------------------------------------------- workspace
    def _poisoned(self, ws_mode):
        ws = self.vae._workspace(self.B, ws_mode)
        ws.fill_(0xFF)
        return ws

    def _views(self, ws_mode):
        offs = (C.c_int64 * len(BUFFERS))()
        n = self.lib.cpb_debug_vae_buffer_offsets(self.B, self.ct, self.z, ws_mode, offs, len(BUFFERS))
        assert n == len(BUFFERS)
        ws = self.vae._ws[ws_mode]
        B, zp = self.B, self.zp
        shapes = {"xp": (B, 80, 160, 4), "a1": (B, 39, 79, 32), "a2": (B, 18, 38, 64), "a3": (B, 8, 18, 128),
                  "a4": (B, 3, 8, 256), "heads": (2, B, zp), "z": (B, zp), "d1": (B, 3, 8, 256), "b1": (B, 8, 18, 128),
                  "b2": (B, 18, 38, 64), "b3": (B, 39, 79, 32), "logits_p": (B, 80, 160, 4), "gz": (B, zp),
                  "gheads": (2, B, zp)}
        out = {}
        for name, o in zip(BUFFERS, offs):
            if name in shapes and o >= 0:
                cnt = int(np.prod(shapes[name]))
                out[name] = ws[o:o + 4 * cnt].view(torch.float32).view(shapes[name])
        out["g"] = {"gA": ws[offs[BUFFERS.index("gA")]:], "gB": ws[offs[BUFFERS.index("gB")]:]} if offs[12] >= 0 else {}
        return out

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
    def forward(self):
        from carla_ppo_b200 import _lib
        self._poisoned(_lib.WS_FORWARD)
        self.losses = self.vae.forward_device(self.x, self.y, self.eps)["losses"]
        torch.cuda.synchronize()
        v = self._views(_lib.WS_FORWARD)
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        relu = torch.relu

        def conv(name, src, tc, k=None):
            def ref(dt, f0, f1):
                s = op(v[src], tc, dt, f0, f1)
                if src == "xp":
                    s = s[..., :3]
                return relu(R.gather(s, wt("encoder/%s/kernel" % name, tc, dt)) + self.w["encoder/%s/bias" % name].to(dt))
            return ref

        def deconv(name, src, tc, out_hw, act=True):
            def ref(dt, f0, f1):
                s = op(v[src], tc, dt, f0, f1)
                r = R.scatter(s, wt("decoder/%s/kernel" % name, tc, dt), out_hw) + self.w["decoder/%s/bias" % name].to(dt)
                return relu(r) if act else r
            return ref

        check_frames(j, "conv1.fwd", v["a1"], conv("conv1", "xp", False), self.frames)
        check_frames(j, "conv2.fwd", v["a2"], conv("conv2", "a1", True), self.frames)
        check_frames(j, "conv3.fwd", v["a3"], conv("conv3", "a2", True), self.frames)
        check_frames(j, "conv4.fwd", v["a4"], conv("conv4", "a3", True), self.frames)

        def heads(i):
            kn, bn = ("mean/kernel", "mean/bias") if i == 0 else ("logstd_sqare/kernel", "logstd_sqare/bias")
            return lambda dt, f0, f1: op(v["a4"], False, dt, f0, f1).reshape(f1 - f0, -1) @ wt(kn, False, dt) + self.w[bn].to(dt)
        check_frames(j, "heads.fwd (mean)", v["heads"][0, :, :z], heads(0), self.frames)
        check_frames(j, "heads.fwd (logstd_sq)", v["heads"][1, :, :z], heads(1), self.frames)
        if not bool((v["heads"][:, :, z:] == 0).all()):
            j.failures.append("heads.fwd %s: padded columns are not 0" % j.tag)

        check_frames(j, "dense1.fwd", v["d1"], lambda dt, f0, f1: (
            R.dense1_fwd(op(v["z"], False, dt, f0, f1), wt("decoder/dense1/kernel", False, dt))
            + self.w["decoder/dense1/bias"].to(dt)).reshape(f1 - f0, 3, 8, 256), self.frames)
        check_frames(j, "deconv1.fwd", v["b1"], deconv("deconv1", "d1", True, (8, 18)), self.frames)
        check_frames(j, "deconv2.fwd", v["b2"], deconv("deconv2", "b1", True, (18, 38)), self.frames)
        check_frames(j, "deconv3.fwd", v["b3"], deconv("deconv3", "b2", True, (39, 79)), self.frames)
        check_frames(j, "deconv4.fwd", v["logits_p"][..., :self.ct], deconv("deconv4", "b3", False, (80, 160), act=False), self.frames)

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
        j, B, k = self.j, self.B, self.w[prefix + "/kernel"].shape[0]
        check_reduction(j, name + ".wgrad", grads[prefix + "/kernel"],
                        lambda dt, f0, f1: R.wgrad(*wgrad_ops(dt, f0, f1), k), self.frames, taps=True)
        check_reduction(j, name + ".bias", grads[prefix + "/bias"],
                        lambda dt, f0, f1: gin[f0:f1].to(dt).sum((0, 1, 2)), self.frames, taps=False)
        if dgrad is not None and self.dgrad:
            check_frames(j, name + ".dgrad", dgrad[0], dgrad[1], self.frames)

    def _group_deconv4(self, v, grads):
        ct, op, wt, B = self.ct, self._op, self._wt, self.B
        dlog = v["logits_p"][..., :ct]
        gA = self._grad_view(v["g"]["gA"], (B, 39, 79, 32))
        self.j.finite("deconv4 input gradient", dlog)
        self._conv_group(grads, "deconv4", "decoder/deconv4", dlog,
                         lambda dt, f0, f1: (op(dlog, False, dt, f0, f1), op(v["b3"], False, dt, f0, f1)),
                         (gA, lambda dt, f0, f1: R.gather(op(dlog, False, dt, f0, f1), wt("decoder/deconv4/kernel", False, dt))
                          * (v["b3"][f0:f1] > 0)))

    def _deconv_group(self, v, grads, name, gin_name, gin_shape, below, out_name, out_shape, masked):
        op, wt, B = self._op, self._wt, self.B
        gin = self._grad_view(v["g"][gin_name], gin_shape)
        out = self._grad_view(v["g"][out_name], out_shape)
        self.j.finite(name + " input gradient", gin)

        def dref(dt, f0, f1):
            r = R.gather(op(gin, True, dt, f0, f1), wt("decoder/%s/kernel" % name, True, dt))
            return r * (v[below][f0:f1] > 0) if masked else r
        self._conv_group(grads, name, "decoder/" + name, gin,
                         lambda dt, f0, f1: (op(gin, True, dt, f0, f1), op(v[below], True, dt, f0, f1)), (out, dref))

    def _group_deconv3(self, v, grads):
        self._deconv_group(v, grads, "deconv3", "gA", (self.B, 39, 79, 32), "b2", "gB", (self.B, 18, 38, 64), True)

    def _group_deconv2(self, v, grads):
        self._deconv_group(v, grads, "deconv2", "gB", (self.B, 18, 38, 64), "b1", "gA", (self.B, 8, 18, 128), True)

    def _group_deconv1(self, v, grads):
        self._deconv_group(v, grads, "deconv1", "gA", (self.B, 8, 18, 128), "d1", "gB", (self.B, 3, 8, 256), False)

    def _group_dense1(self, v, grads):
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        gin = self._grad_view(v["g"]["gB"], (B, 6144))
        j.finite("dense1 input gradient", gin)
        check_reduction(j, "dense1.wgrad", grads["decoder/dense1/kernel"],
                        lambda dt, f0, f1: op(v["z"], False, dt, f0, f1)[:, :z].T @ gin[f0:f1].to(dt), self.frames, taps=False)
        check_reduction(j, "dense1.bias", grads["decoder/dense1/bias"], lambda dt, f0, f1: gin[f0:f1].to(dt).sum(0), self.frames, taps=False)
        if self.dgrad:
            check_frames(j, "dense1.dgrad", v["gz"][:, :z],
                         lambda dt, f0, f1: gin[f0:f1].to(dt) @ wt("decoder/dense1/kernel", False, dt).T, self.frames)
        if not bool((v["gz"][:, z:] == 0).all()):
            j.failures.append("dense1.dgrad %s: padded columns of gz are not 0" % j.tag)

    def _group_heads(self, v, grads):
        j, B, z, op, wt = self.j, self.B, self.z, self._op, self._wt
        gh = v["gheads"]
        j.finite("heads input gradient", gh[:, :, :z])
        a4 = v["a4"].reshape(B, -1)
        for i, name in enumerate(("mean", "logstd_sqare")):
            check_reduction(j, "heads.wgrad (%s)" % name, grads[name + "/kernel"],
                            lambda dt, f0, f1, i=i: a4[f0:f1].to(dt).T @ gh[i, f0:f1, :z].to(dt), self.frames, taps=False)
            check_reduction(j, "heads.bias (%s)" % name, grads[name + "/bias"],
                            lambda dt, f0, f1, i=i: gh[i, f0:f1, :z].to(dt).sum(0), self.frames, taps=False)
        out = self._grad_view(v["g"]["gA"], (B, 3, 8, 256))
        if self.dgrad:
            check_frames(j, "heads.dgrad", out, lambda dt, f0, f1: (
            R.heads_dgrad(gh[:, f0:f1].to(dt), wt("mean/kernel", False, dt), wt("logstd_sqare/kernel", False, dt))
            .reshape(f1 - f0, 3, 8, 256) * (v["a4"][f0:f1] > 0)), self.frames)

    def _enc_group(self, v, grads, name, gin_name, gin_shape, src, out_name, out_shape):
        op, wt, B = self._op, self._wt, self.B
        gin = self._grad_view(v["g"][gin_name], gin_shape)
        out = self._grad_view(v["g"][out_name], out_shape)
        self.j.finite(name + " input gradient", gin)
        self._conv_group(grads, name, "encoder/" + name, gin,
                         lambda dt, f0, f1: (op(v[src], True, dt, f0, f1), op(gin, True, dt, f0, f1)),
                         (out, lambda dt, f0, f1: R.scatter(op(gin, True, dt, f0, f1), wt("encoder/%s/kernel" % name, True, dt),
                                                            out_shape[1:3]) * (v[src][f0:f1] > 0)))

    def _group_conv4(self, v, grads):
        self._enc_group(v, grads, "conv4", "gA", (self.B, 3, 8, 256), "a3", "gB", (self.B, 8, 18, 128))

    def _group_conv3(self, v, grads):
        self._enc_group(v, grads, "conv3", "gB", (self.B, 8, 18, 128), "a2", "gA", (self.B, 18, 38, 64))

    def _group_conv2(self, v, grads):
        # the whole pass: conv2's group, then conv1's weight and bias gradient from conv2's output gradient
        B, op = self.B, self._op
        self._enc_group(v, grads, "conv2", "gA", (B, 18, 38, 64), "a1", "gB", (B, 39, 79, 32))
        gin = self._grad_view(v["g"]["gB"], (B, 39, 79, 32))
        self._conv_group(grads, "conv1", "encoder/conv1", gin,
                         lambda dt, f0, f1: (op(v["xp"], False, dt, f0, f1)[..., :3], op(gin, False, dt, f0, f1)))


@pytest.mark.parametrize("mode", MODES, ids=["simt", "tc3xtf32", "tf32"])
@pytest.mark.parametrize("batch,ct,z", CASES, ids=["B%d-ct%d-z%d" % c for c in CASES])
def test_every_layer_pass_on_the_devices_own_operands(lib, tmp_path, mode, batch, ct, z):
    case = Case(lib, tmp_path, mode, batch, ct, z)
    case.forward()
    case.backward()
    print("\n%s: worst err/gate %s" % (case.j.tag, ", ".join("%s %.2f" % kv for kv in sorted(case.j.worst.items(), key=lambda kv: -kv[1])[:6])))
    assert not case.j.failures, "\n".join(case.j.failures[:40])


def test_the_stop_hook_changes_nothing_when_unset(lib, tmp_path):
    """Setting a stop and clearing it again leaves loss_grad bit-identical with the same launch count."""
    from carla_ppo_b200 import _lib
    case = Case(lib, tmp_path, 1, 33, 3, 64)
    res = []
    for stop in (None, b"heads.dgrad", None):
        _lib.check(lib.cpb_debug_vae_backward_stop(stop))
        lib.cpb_reset_launch_count()
        case.vae.loss_grad_device(case.x, case.y, case.eps)
        torch.cuda.synchronize()
        res.append((case.vae.grads.clone(), case.vae._losses.clone(), lib.cpb_launch_count()))
    assert torch.equal(res[0][0], res[2][0]) and torch.equal(res[0][1], res[2][1]) and res[0][2] == res[2][2]
    assert res[1][2] < res[0][2] and not torch.equal(res[0][0], res[1][0])
    # a rejected name leaves the stop as it was: still the whole pass
    assert lib.cpb_debug_vae_backward_stop(b"conv1.dgrad") == -1
    case.vae.loss_grad_device(case.x, case.y, case.eps)
    assert torch.equal(case.vae.grads, res[0][0])
