"""Per-tensor gradient error of one ConvVAE step against the float64 oracle (diagnostic for __graft_entry__.smoke())."""
import os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from carla_ppo_b200.vae.models import ConvVAE
from oracle import vae_oracle as vo, torch_ref

def rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return np.linalg.norm(a - b) / np.linalg.norm(b)

seed, B = int(os.environ.get("SEED", "0")), int(os.environ.get("B", "4"))
w = vo.glorot_init(0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.environ.get("WEIGHTS") == "shipped":
    zv = np.load(os.path.join(ROOT, "tests", "golden", "vae_rgb_ckpt232.npz"))
    w = {k: zv[k] for k in vo.param_shapes().keys()}
vae = ConvVAE((80, 160, 3), z_dim=64, loss_fn="mse", model_dir=tempfile.mkdtemp(), seed=0)
vae.init_session(init_logging=False)
vae.set_weights(w)
x = np.random.RandomState(seed).rand(B, 80, 160, 3).astype(np.float32)
if os.environ.get("FRAMES") == "shipped":
    x = (np.load(os.path.join(ROOT, "tests", "golden", "frames_u8.npz"))["rgb"][seed:seed + B] / np.float32(255.0)).astype(np.float32)
eps = np.random.RandomState(seed + 1).randn(B, 64).astype(np.float32)
vae.train_step(x, x, eps)
p64 = {k: v.astype(np.float64) for k, v in w.items()}
ref = vo.loss_and_grads(p64, x, x, eps)
g32 = torch_ref.vae_loss_and_grads(w, x, x, eps, dtype=torch.float32)["grads"]
got = vae.get_grads()
print("seed %d B %d" % (seed, B))
for k in p64:
    d = np.abs(got[k].astype(np.float64) - ref["grads"][k])
    print("  %-26s gpu %.2e  cpu32 %.2e   max|d| %.2e at %s (|g| there %.2e, max|g| %.2e)" % (
        k, rel(got[k], ref["grads"][k]), rel(g32[k], ref["grads"][k]), d.max(), np.unravel_index(d.argmax(), d.shape),
        abs(ref["grads"][k].ravel()[d.argmax()]), np.abs(ref["grads"][k]).max()))
