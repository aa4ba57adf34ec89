"""Per-tensor parameter error after 3 Adam steps from the shipped weights (the single-rank half of scripts/dp_check.py).
MODE=ref (CPU): float64 oracle + float32 CPU restatement -> scripts/_diag_ref.npz;  MODE=gpu: compare the device against it."""
import os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import vae_oracle as vo

B = int(os.environ.get("B", "128"))
zv = np.load(os.path.join(ROOT, "tests", "golden", "vae_rgb_ckpt232.npz"))
w0 = {k: zv[k] for k in vo.param_shapes().keys()}
x = np.random.RandomState(0).rand(B, 80, 160, 3).astype(np.float32)
eps = np.random.RandomState(1).randn(B, 64).astype(np.float32)
ref_path = os.path.join(ROOT, "scripts", "_diag_ref_B%d.npz" % B)

def rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))

if os.environ.get("MODE", "gpu") == "ref":
    from oracle.torch_ref import TorchVAETrainer
    p64 = {k: v.astype(np.float64) for k, v in w0.items()}
    st = vo.adam_init_state(p64)
    g1 = vo.loss_and_grads({k: v.astype(np.float64) for k, v in w0.items()}, x, x, eps)["grads"]
    cpu32 = TorchVAETrainer(w0, lr=1e-4, loss_type="mse")
    for step in range(3):
        vo.train_step(p64, st, x, x, eps, lr=1e-4)
        cpu32.step(torch.from_numpy(x), torch.from_numpy(x), torch.from_numpy(eps))
    out = {}
    for k in p64:
        out["p64/" + k] = p64[k]; out["p32/" + k] = cpu32.p[k].detach().numpy(); out["g1/" + k] = g1[k]
    np.savez(ref_path, **out)
    print("wrote", ref_path)
else:
    from carla_ppo_b200.vae.models import ConvVAE
    r = np.load(ref_path)
    vae = ConvVAE((80, 160, 3), z_dim=64, loss_fn="mse", model_dir=tempfile.mkdtemp(), seed=0)
    vae.init_session(init_logging=False)
    vae.set_weights(w0)
    xd, ed = torch.tensor(x, device="cuda"), torch.tensor(eps, device="cuda")
    vae.train_step_device(xd, xd, ed)
    g = vae.get_grads()
    for _ in range(2):
        vae.train_step_device(xd, xd, ed)
    got = vae.get_weights()
    print("B %d" % B)
    for k in w0:
        d = np.abs(got[k].astype(np.float64) - r["p64/" + k])
        print("  %-26s params gpu %.2e cpu32 %.2e | first grad gpu %.2e | max|dp| %.2e (lr=1e-4) n=%d" % (
            k, rel(got[k], r["p64/" + k]), rel(r["p32/" + k], r["p64/" + k]), rel(g[k], r["g1/" + k]), d.max(), d.size))
