"""GPU parity at the sizes that SHIP: BASELINE configs[1] (one 4096-frame batch on one GPU) and the 512-frame shard
one rank of configs[3] executes, against the float64 golden vectors of tests/golden/make_golden_large.py.

Tile scheduling (super-tile counts, m-groups, split-K factors) depends on the batch, so the small-batch oracle tests
do not cover these launches.  Every gate is max(1e-5, 2 x the error the float32 CPU restatement of the reference graph
makes on the same inputs) -- the float32 error is stored in the golden file next to each quantity (err32*).
"""
import os

import numpy as np
import pytest

from harness import conv_workspace, lib, library_state, make_conv_vae, math_mode  # noqa: F401
from helpers import GOLDEN, rel_l2, shipped_vae_weights

pytestmark = pytest.mark.gpu

TOL = 1e-5


def large_inputs(n):
    """Regenerates the inputs of make_golden_large.py (630 MB at n = 4096: only the outputs are committed)."""
    x = np.random.RandomState(4096).rand(4096, 80, 160, 3).astype(np.float32)[:n]
    eps = np.random.RandomState(4097).randn(4096, 64).astype(np.float32)[:n]
    return x, eps


@pytest.mark.parametrize("batch", [512, 4096])
@pytest.mark.parametrize("mode", [1, 0], ids=["tc3xtf32", "simt"])
def test_shipping_batch_matches_float64_golden(tmp_path, lib, batch, mode):
    import torch
    from carla_ppo_b200 import _lib
    if mode == 0 and batch == 4096:
        pytest.skip("the fp32 SIMT path is the fallback arithmetic; its batch-dependent scheduling is covered at 512")
    g = np.load(os.path.join(GOLDEN, "large_B%d.npz" % batch))
    with math_mode(lib, mode):
        w = shipped_vae_weights()[0]
        vae = make_conv_vae(tmp_path, w)
        x, eps = large_inputs(batch)
        xd = torch.from_numpy(x).to(vae._device); ed = torch.from_numpy(eps).to(vae._device)
        vae.loss_grad_device(xd, xd, ed)
        vae._check_flags()
        losses = vae._losses.cpu().numpy().astype(np.float64)
        assert abs(losses[0] - g["recon"]) / g["recon"] < max(TOL, 2 * float(g["err32_recon"]))
        assert abs(losses[1] - g["kl"]) / g["kl"] < TOL
        # per-frame forward quantities of the sampled frames
        view = conv_workspace(vae, batch, _lib.WS_TRAIN)
        idx = torch.from_numpy(g["sample_idx"]).to(vae._device)
        heads = view["heads"]
        assert rel_l2(heads[0].index_select(0, idx).cpu().numpy(), g["mean"]) < max(TOL, 2 * float(g["err32_mean"]))
        assert rel_l2(heads[1].index_select(0, idx).cpu().numpy(), g["logvar"]) < max(TOL, 2 * float(g["err32_logvar"]))
        fl = view["frame_loss"].index_select(0, idx).cpu().numpy()
        assert rel_l2(fl, g["frame_recon"]) < max(TOL, 2 * float(g["err32_frame_recon"]))
        kr = view["kl_rows"].index_select(0, idx).cpu().numpy()
        assert rel_l2(kr, g["frame_kl"]) < TOL
        # the full-batch gradient, every tensor (large ones on the committed fixed-stride subsample)
        got = vae.get_grads()
        for name in w:
            ref = g["grad/" + name]
            mine = got[name].ravel()[g["gidx/" + name]]
            err = np.linalg.norm(mine.astype(np.float64) - ref) / np.linalg.norm(ref)
            gate = max(TOL, 2 * float(g["err32/" + name]))
            assert err < gate, "%s: rel err %.3e, gate %.3e (fp32 CPU restatement %.3e)" % (name, err, gate, float(g["err32/" + name]))
