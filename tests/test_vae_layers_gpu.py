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
import pytest
import torch

from harness import fp32_matmul, lib, library_state, math_mode  # noqa: F401
from layer_judge import Case

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("fp32_matmul")]      # err_f32: plain SGEMM

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


@pytest.mark.parametrize("mode", MODES, ids=["simt", "tc3xtf32", "tf32"])
@pytest.mark.parametrize("batch,ct,z", CASES, ids=["B%d-ct%d-z%d" % c for c in CASES])
def test_every_layer_pass_on_the_devices_own_operands(lib, tmp_path, mode, batch, ct, z):
    with math_mode(lib, mode):
        case = Case(lib, tmp_path, mode, batch, ct, z)
        case.forward()
        case.backward()
    case.j.report()


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
