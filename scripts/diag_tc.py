"""GPU diagnostics for the wgmma 3xTF32 kernel: dense GEMM error vs fp64 as a function of K and data
statistics, and per-buffer differences between math mode 0 (SIMT) and 1 (tensor core) after a VAE forward."""
import os, sys, ctypes as C, tempfile
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from carla_ppo_b200 import _lib
lib = _lib.load()

def gemm(a, bt):
    m, k = a.shape; n = bt.shape[0]
    ta = torch.tensor(a, device="cuda"); tb = torch.tensor(bt, device="cuda")
    d = torch.empty(m, n, device="cuda"); sc = torch.empty(2 * n * k + m * k, device="cuda")
    _lib.check(lib.cpb_debug_tc_gemm(ta.data_ptr(), tb.data_ptr(), d.data_ptr(), m, n, k, sc.data_ptr(), _lib.current_stream_handle()))
    torch.cuda.synchronize()
    return d.cpu().numpy()

rs = np.random.RandomState(0)
print("dense D = A Bt^T: rel_l2 error vs fp64, mean signed rel error (bias), fp32-numpy error")
for (m, n, k, kind) in [(256, 128, 32, "randn"), (256, 128, 256, "randn"), (256, 128, 1024, "randn"), (256, 128, 4096, "randn"),
                        (256, 128, 1024, "pos"), (256, 128, 4096, "pos"), (300, 64, 800, "randn"), (300, 32, 576, "randn"), (256, 256, 2048, "randn"),
                        (256, 128, 1024, "relu")]:
    if kind == "randn": a = rs.randn(m, k); bt = rs.randn(n, k)
    elif kind == "pos": a = rs.rand(m, k); bt = rs.rand(n, k)
    else: a = np.maximum(rs.randn(m, k), 0); bt = rs.randn(n, k)
    a = a.astype(np.float32); bt = bt.astype(np.float32)
    ref = a.astype(np.float64) @ bt.astype(np.float64).T
    got = gemm(a, bt)
    f32 = a @ bt.T
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    bias = np.mean((got - ref) / np.where(np.abs(ref) > 1e-3 * np.abs(ref).max(), ref, np.inf))
    print("  M=%d N=%d K=%d %-5s  tc_err=%.2e bias=%+.2e   numpy_f32_err=%.2e" % (m, n, k, kind, err, bias, np.linalg.norm(f32 - ref) / np.linalg.norm(ref)))

# per-buffer comparison of the two math modes
from helpers import shipped_vae_weights
from carla_ppo_b200.vae.models import ConvVAE
w = shipped_vae_weights()[0]
names = ["xp", "a1", "a2", "a3", "a4", "heads", "z", "d1", "b1", "b2", "b3", "logits_p", "gA", "gB"]
B = 16
offs = (C.c_int64 * 16)()
n = lib.cpb_debug_vae_buffer_offsets(B, 3, 64, 1, offs, 16)
sizes = {"a1": B*39*79*32, "a2": B*18*38*64, "a3": B*8*18*128, "a4": B*6144, "heads": 2*B*64, "d1": B*6144, "b1": B*8*18*128, "b2": B*18*38*64, "b3": B*39*79*32, "logits_p": B*12800*4}
x = np.random.RandomState(0).rand(B, 80, 160, 3).astype(np.float32); eps = np.random.RandomState(1).randn(B, 64).astype(np.float32)
snap = {}
for mode in (0, 1):
    _lib.check(lib.cpb_set_math_mode(mode))
    vae = ConvVAE((80,160,3), z_dim=64, loss_fn="mse", model_dir=tempfile.mkdtemp(), seed=0); vae.init_session(init_logging=False); vae.set_weights(w)
    xd = torch.tensor(x, device="cuda"); ed = torch.tensor(eps, device="cuda")
    vae.forward_device(xd, xd, ed)
    torch.cuda.synchronize()
    ws = vae._ws[_lib.WS_FORWARD]
    snap[mode] = {nm: ws[offs[i]:offs[i] + 4*sizes[nm]].view(torch.float32).clone().cpu().numpy().astype(np.float64) for i, nm in enumerate(names[:n]) if nm in sizes}
print("forward buffers, shipped weights B=16: ||tc - simt|| / ||simt||, mean signed rel diff")
for nm in sizes:
    a, b = snap[1][nm], snap[0][nm]
    big = np.abs(b) > 1e-2 * np.abs(b).max()
    print("  %-9s %.2e   bias %+.2e" % (nm, np.linalg.norm(a - b) / np.linalg.norm(b), np.mean((a[big] - b[big]) / b[big])))
