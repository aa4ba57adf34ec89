"""Both VAEs at the largest batches they accept: the tensor-core offset bound of math modes 1 and 2 (B * H1 * W1 * 32 <
2^31 for the ConvVAE; B * 38400 < 2^31 for the MlpVAE's five frame-wide products in mode 2) and, in math mode 0, past
2^31 elements, where the kernels index in 64 bits.

Placed-frame batches (tests/large_batch.py): all but a few frames are null frames that compute exactly 0, and the live
frames sit on both sides of every 2^29 .. 2^32 element boundary of every checked buffer.  Each case fills the workspace
with NaN bytes before every call, and checks that
  * every checked buffer is exactly 0 on every null frame and finite on every live frame (a write that lands in the
    wrong frame, or a missed write that leaves NaN behind, fails here);
  * every layer pass on the device's own operands of the live frames matches float64 at tests/test_vae_layers_gpu.py's
    gates (tests/test_mlp_depth_gpu.py's for the MlpVAE).  Null operands are exactly 0, so the weight- and bias-gradient
    references summed over the live frames alone are exact; both losses are the live frames' sums / B;
  * the encoding of the live frames is bit-identical to the same frames encoded as a batch of their own (for the MlpVAE
    at 55 925 frames in mode 2: in mode 1, which shows the call took the fp32 path);
  * every call returns CPB_OK (the models raise otherwise).
Full-batch accuracy: the ConvVAE at 80x160 with every frame random, in mode 1 at the bound and in mode 0 above it -- all
22 weight and bias gradients (reductions over every frame) and both losses against float64 in frame chunks.

One workspace is alive at a time.  A case that the card cannot hold skips, naming the bytes it needs and the bytes free."""
import contextlib

import numpy as np
import pytest
import torch

import large_batch as LB
import vae_checks as VC
from harness import fp32_matmul, lib, library_state, make_mlp, math_mode, mlp_relu_masks, mlp_workspace  # noqa: F401
from helpers import rel_l2
from layer_judge import Case, Judge, spans

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("fp32_matmul")]      # err_f32: plain SGEMM

REF_BYTES = 4 << 30          # the float64 reference chunks and per-frame reductions (deconv3's data-gradient im2col: 1.1 GB)
LOSS_FLOOR = 1e-5            # the loss floor of tests/test_vae_gpu.py and tests/test_mlp_depth_gpu.py


@pytest.fixture(autouse=True)
def free_memory():
    yield
    torch.cuda.empty_cache()


def need_memory(case, mode, extra):
    """Skip unless the card holds the case's largest workspace in `mode`, its inputs and REF_BYTES."""
    need = case["bytes"][mode] + extra + REF_BYTES
    free = torch.cuda.mem_get_info()[0]
    if need > free:
        pytest.skip("needs %d bytes of device memory, %d free" % (need, free))


def placed_inputs(batch, hw, ct, z, live, seed):
    """u8 source 0, f32 target 0.5 and eps 0 on the null frames; random data on the live ones."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    idx = torch.tensor(live, device="cuda")
    n, (h, w) = len(live), hw
    x = torch.zeros(batch, h, w, 3, dtype=torch.uint8, device="cuda")
    x[idx] = torch.randint(0, 256, (n, h, w, 3), generator=g, device="cuda", dtype=torch.uint8)
    y = torch.full((batch, h, w, ct), 0.5, device="cuda")
    y[idx] = torch.rand(n, h, w, ct, generator=g, device="cuda")
    eps = torch.zeros(batch, z, device="cuda")
    eps[idx] = torch.randn(n, z, generator=g, device="cuda")
    return x, y, eps


def input_bytes(batch, hw, ct=3, z=64):
    return batch * hw[0] * hw[1] * (3 + 4 * ct) + 4 * batch * z


def free_workspaces(vae):
    vae._ws.clear()
    torch.cuda.empty_cache()


def check_losses(case, losses, v, floor=LOSS_FLOOR):
    """The MSE and KL of a forward call against float64 on its own logits and heads, summed over spans(case.frames) / B."""
    j, z, ct = case.j, case.z, case.ct
    r = {torch.float64: [0.0, 0.0], torch.float32: [0.0, 0.0]}
    for f0, f1 in spans(case.frames):
        for dt in r:
            lg = v["logits_p"][f0:f1, ..., :ct].to(dt)
            m, lv = v["heads"][0, f0:f1, :z].to(dt), v["heads"][1, f0:f1, :z].to(dt)
            r[dt][0] = r[dt][0] + ((case.y[f0:f1].to(dt) - torch.sigmoid(lg)) ** 2).sum()
            r[dt][1] = r[dt][1] + -0.5 * (1.0 + lv - m * m - torch.exp(lv)).sum()
    for i, name in enumerate(("recon", "kl")):
        r64, r32 = r[torch.float64][i] / case.B, r[torch.float32][i].double() / case.B
        j.gate("loss (%s)" % name, "value", (losses[i].double() - r64) ** 2, (r32 - r64) ** 2, r64 * r64, floor)


def encode_invariance(j, vae, x, live, small_mode=None):
    """mean and logvar of the live frames: bit-identical to the same frames encoded as their own batch (in small_mode,
    if given)."""
    mean, logvar = vae.encode_device(x, return_logvar=True)
    mean, logvar = mean[live], logvar[live]
    free_workspaces(vae)
    with contextlib.nullcontext() if small_mode is None else math_mode(vae._libh, small_mode):
        sm, sl = vae.encode_device(x[live].contiguous(), return_logvar=True)
    free_workspaces(vae)
    for what, a, b in (("mean", mean, sm), ("logvar", logvar, sl)):
        if not torch.equal(a, b):
            rows = [live[i] for i in torch.nonzero((a != b).any(1))[:, 0].tolist()]
            j.failures.append("encode %s %s: frames %s differ from the same frames encoded on their own" % (what, j.tag, rows))


# --------------------------------------------------------------------------------------------------- ConvVAE, placed frames
def place(case, live, hw):
    """Make a layer-test case a placed-frame batch: every bias 0, null frames everywhere but `live`."""
    for k in case.w:
        if k.endswith("bias"):
            case.w[k].zero_()
    case.vae.set_weights({k: v.cpu().numpy() for k, v in case.w.items()})
    case.x = case.y = case.eps = None
    torch.cuda.empty_cache()
    case.x, case.y, case.eps = placed_inputs(case.B, hw, case.ct, case.z, live, 77 + case.B)
    case.frames = [(f, f + 1) for f in live]
    case.j.live = live


CONV = [("conv80x160-bound", 1), ("conv80x160-bound", 2), ("conv80x160-simt", 0),
        ("conv512x512-bound", 1), ("conv512x512-bound", 2), ("conv512x512-simt", 0)]


@pytest.mark.parametrize("name,mode", CONV, ids=["%s-mode%d" % c for c in CONV])
def test_conv_vae_placed_frames(lib, tmp_path, name, mode):
    from carla_ppo_b200 import _lib
    spec = LB.CASES[name]
    hw, batch = spec["hw"], spec["batch"]
    need_memory(spec, mode, input_bytes(batch, hw) + 4 * batch * hw[0] * hw[1] * 3)     # + the case's own f32 frames
    live = LB.live_frames(batch, LB.conv_counts(*hw))
    with math_mode(lib, mode):
        case = Case(lib, tmp_path, mode, batch, 3, 64, None if hw == (80, 160) else hw)
        case.j.tag = "%s %s" % (name, case.j.tag)
        place(case, live, hw)
        encode_invariance(case.j, case.vae, case.x, live)
        encode_only = spec["ws"] == _lib.WS_ENCODE
        if encode_only:
            case.forward(encode_only=True)          # an encode call (the 512x512 case above the bound)
        else:
            case.forward()
        v = case._views(_lib.WS_ENCODE if encode_only else _lib.WS_FORWARD)
        for nm in ("xp", "z"):
            if nm in v:
                case.j.zeros(nm, v[nm])
        case.j.zeros("heads", v["heads"].transpose(0, 1))
        if not encode_only:
            check_losses(case, case.losses, v)
        del v
        free_workspaces(case.vae)
        if spec["ws"] == _lib.WS_TRAIN:
            case.backward()
            free_workspaces(case.vae)
        case.j.report()


# --------------------------------------------------------------------------------------------------- ConvVAE, every frame
FULL = [("conv80x160-bound", 1), ("conv80x160-simt", 0)]


@pytest.mark.parametrize("name,mode", FULL, ids=["%s-mode%d" % c for c in FULL])
def test_conv_vae_reductions_over_the_whole_batch(lib, tmp_path, name, mode):
    """Every weight and bias gradient and both losses at B = 21 781 (mode 1) and 22 000 (mode 0), every frame random,
    against float64 in frame chunks at max(2e-6, 2 x err_f32): the accumulation length along the batch axis."""
    from carla_ppo_b200 import _lib
    spec = LB.CASES[name]
    batch = spec["batch"]
    need_memory(spec, mode, input_bytes(batch, (80, 160)) + 4 * batch * 80 * 160 * 3)
    with math_mode(lib, mode):
        case = Case(lib, tmp_path, mode, batch, 3, 64)
        case.j.tag = "%s every frame %s" % (name, case.j.tag)
        case.dgrad = False
        case._poisoned(_lib.WS_FORWARD)
        losses = case.vae.forward_device(case.x, case.y, case.eps)["losses"]
        torch.cuda.synchronize()
        check_losses(case, losses, case._views(_lib.WS_FORWARD))
        free_workspaces(case.vae)
        case.backward()
        free_workspaces(case.vae)
        case.j.report()


# --------------------------------------------------------------------------------------------------- MlpVAE, placed frames
MLP = [("mlp-last-tc", 2), ("mlp-first-fp32", 0), ("mlp-first-fp32", 1), ("mlp-first-fp32", 2), ("mlp-8192-last-tc", 2)]


@pytest.mark.parametrize("name,mode", MLP, ids=["%s-mode%d" % c for c in MLP])
def test_mlp_vae_placed_frames(lib, tmp_path, name, mode):
    import mlp_depth_oracle as mdo
    from carla_ppo_b200 import _lib
    from oracle import vae_oracle as vo
    from tf32_oracle import round_tf32
    spec = LB.CASES[name]
    (enc, dec), batch = spec["mlp"], spec["batch"]
    need_memory(spec, mode, input_bytes(batch, (80, 160)))
    with math_mode(lib, mode):
        tc = mode == 2 and batch * VC.IN < 1 << 31
        j = Judge("%s mode %d B=%d" % (name, mode, batch))
        live = LB.live_frames(batch, LB.mlp_counts(enc, dec))
        j.live = live
        w = mdo.glorot_init(1, encoder_sizes=enc, decoder_sizes=dec)          # every bias 0
        vae = make_mlp(tmp_path, w, enc, dec, loss="mse")
        x, y, eps = placed_inputs(batch, (80, 160), 3, 64, live, 5 + batch)
        full = name != "mlp-8192-last-tc"
        widths = {"x": VC.IN, "logits": VC.IN}
        widths.update({"h%d" % i: v for i, v in enumerate(enc)})
        widths.update({"g%d" % k: v for k, v in enumerate(dec)})

        def zeros(ws_mode, extra=()):
            t = mlp_workspace(vae, batch, ws_mode, dict(widths, **dict(extra)), host=False)
            for nm, v in t.items():
                j.zeros(nm, v)

        if full:
            encode_invariance(j, vae, x, live, small_mode=1 if mode == 2 and not tc else None)
            vae._workspace(batch, _lib.WS_FORWARD).fill_(0xFF)
            out = vae.forward_device(x, y, eps, want_latents=True)
            torch.cuda.synchronize()
            zeros(_lib.WS_FORWARD)
            fwd = {k: out[k][live].cpu().numpy().astype(np.float64) for k in ("mean", "logvar")}
            fwd_losses = out["losses"].cpu().numpy().astype(np.float64)
            if tc:
                for what, err in VC.forward_products(vae, w, batch, live).items():
                    if not err < VC.UNIT_TOL:
                        j.failures.append("%s %s: rel err %.3e on the live frames" % (what, j.tag, err))
            free_workspaces(vae)
        vae._workspace(batch, _lib.WS_TRAIN).fill_(0xFF)
        vae.grads.fill_(float("nan"))
        vae.loss_grad_device(x, y, eps)
        torch.cuda.synchronize()
        zeros(_lib.WS_TRAIN, {"gb": enc[0]})
        got = vae.get_grads()
        losses = vae._losses.cpu().numpy().astype(np.float64)
        masks = mlp_relu_masks(vae, batch, live)
        xl = mlp_workspace(vae, batch, _lib.WS_TRAIN, {"x": VC.IN}, live)["x"].reshape(len(live), 80, 160, 3)
        yl, el = y[live].cpu().numpy(), eps[live].cpu().numpy()
        if tc:
            for what, err in VC.backward_products(vae, w, batch, live).items():
                if not err < VC.UNIT_TOL:
                    j.failures.append("%s %s: rel err %.3e on the live frames" % (what, j.tag, err))
        free_workspaces(vae)
        scale = len(live) / batch               # the device averages over B, the oracle over the live frames
        ref = mdo.loss_and_grads(w, xl, yl, el, "mse", relu_masks=masks)
        approx = (mdo.loss_and_grads(w, xl, yl, el, "mse", relu_masks=masks, tc_round=round_tf32) if tc else
                  mdo.loss_and_grads(w, xl, yl, el, "mse", relu_masks=masks, dtype=np.float32))

        def gate(what, dev, r, a, floor=VC.FWD_TOL):
            err, g = rel_l2(dev, r), max(floor, 2.0 * rel_l2(a, r))
            j.worst[what] = max(j.worst.get(what, 0.0), err / g)
            if not err < g:
                j.failures.append("%s %s: rel err %.3e > gate %.3e" % (what, j.tag, err, g))
        for name_, g in ref["grads"].items():
            gate(name_, got[name_], g * scale, approx["grads"][name_] * scale)
        for i, k in enumerate(("recon", "kl")):
            gate("loss (%s) of loss_grad" % k, losses[i], ref[k] * scale, approx[k] * scale)
        if full:
            for i, k in enumerate(("recon", "kl")):
                gate("loss (%s) of forward" % k, fwd_losses[i], ref[k] * scale, approx[k] * scale)
            for k in ("mean", "logvar"):
                gate(k, fwd[k], ref[k], approx[k])
        j.report()
