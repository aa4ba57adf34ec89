"""The tensor-core tap-GEMM is bit-identical across CPB_TC_CLUSTER (1, the default, and weight multicast over 2 / 4 / 8
CTAs) at the ConvVAE's own layer shapes: gather form, quad scatter form with border taps, N/BN from 1 to 8 and ragged
last m-tiles -- which the dense one-tap GEMMs of test_tc_gpu.py / test_tf32_gpu.py do not reach.  One subprocess per
cluster size (the variable is read once per process) runs cpb_vae_loss_grad at B = 8 in math modes 1 and 2 and hashes
the losses, the gradient and the tensor-core layers' outputs in the workspace."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SNIPPET = r"""
import ctypes as C, hashlib, sys, tempfile
import numpy as np, torch
sys.path.insert(0, %r)
from carla_ppo_b200 import _lib
from carla_ppo_b200.vae.models import ConvVAE
from oracle import vae_oracle as vo
lib = _lib.load()
B = 8
w = vo.glorot_init(0)
vae = ConvVAE(source_shape=(80, 160, 3), z_dim=64, loss_fn="mse", model_dir=tempfile.mkdtemp(), seed=0)
vae.init_session(init_logging=False)
vae.set_weights(w)
x = np.random.RandomState(0).rand(B, 80, 160, 3).astype(np.float32)
eps = np.random.RandomState(1).randn(B, 64).astype(np.float32)
tx, te = torch.as_tensor(x, device=vae._device), torch.as_tensor(eps, device=vae._device)
names = ["xp", "a1", "a2", "a3", "a4", "heads", "z", "d1", "b1", "b2", "b3", "logits_p", "gA", "gB", "frame_loss", "kl_rows"]
sizes = {"a2": 18 * 38 * 64, "a3": 8 * 18 * 128, "a4": 3 * 8 * 256, "b1": 8 * 18 * 128, "b2": 18 * 38 * 64, "b3": 39 * 79 * 32}
offs = (C.c_int64 * len(names))()
lib.cpb_debug_vae_buffer_offsets(B, 3, 64, _lib.WS_TRAIN, offs, len(names))
for mode in (_lib.MATH_3XTF32, _lib.MATH_TF32):
    _lib.check(lib.cpb_set_math_mode(mode))
    vae.loss_grad_device(tx, tx, te)
    torch.cuda.synchronize()
    h = hashlib.sha256()
    h.update(vae._losses.cpu().numpy().tobytes())
    h.update(vae.grads.cpu().numpy().tobytes())
    ws = vae._ws[_lib.WS_TRAIN]
    for nm, cnt in sizes.items():
        o = offs[names.index(nm)]
        h.update(ws[o:o + 4 * B * cnt].cpu().numpy().tobytes())
    print("HASH", mode, h.hexdigest())
    if mode == _lib.MATH_3XTF32:
        ref = vo.loss_and_grads({k: v.astype(np.float64) for k, v in w.items()}, x, x, eps, "mse", want_grads=False)
        print("RECON_ERR", abs(float(vae._losses[0]) - ref["recon"]) / ref["recon"])
"""


def test_vae_layers_are_bit_identical_across_cluster_sizes():
    hashes, errs = {}, {}
    for cs in ("1", "2", "4", "8"):
        env = dict(os.environ, CPB_TC_CLUSTER=cs)
        res = subprocess.run([sys.executable, "-c", _SNIPPET % ROOT], env=env, capture_output=True, text=True,
                             timeout=600, cwd=ROOT)
        assert res.returncode == 0, res.stderr[-2000:]
        out = res.stdout.splitlines()
        hashes[cs] = [ln for ln in out if ln.startswith("HASH")]
        errs[cs] = float([ln for ln in out if ln.startswith("RECON_ERR")][0].split()[1])
        assert len(hashes[cs]) == 2, res.stdout
    assert hashes["1"] == hashes["2"] == hashes["4"] == hashes["8"], hashes
    assert errs["1"] < 1e-5, errs
