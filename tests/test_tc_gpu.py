"""Unit parity of the two tensor-core (wgmma) kernels through their C-ABI debug entries (cpb_debug_tc_gemm /
cpb_debug_tc_wgrad) against float64 NumPy, at shapes that exercise every tile width, ragged row counts, one / many
k-blocks and multi-tile persistence; plus bit-identity of the tap-GEMM across cluster (weight-multicast) sizes.

Tolerance: 3xTF32 with chunked accumulation measures 6e-7 .. 9e-7 norm-wise (scripts/diag_tc.py); the bar here is
2e-6, five times inside the 1e-5 the layer-level tests use."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gemm(a, bt):
    import torch
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    m, k = a.shape
    n = bt.shape[0]
    ta, tb = torch.tensor(a, device="cuda"), torch.tensor(bt, device="cuda")
    d = torch.full((m, n), float("nan"), device="cuda")
    scratch = torch.empty(2 * n * k + m * k, device="cuda")
    _lib.check(lib.cpb_debug_tc_gemm(ta.data_ptr(), tb.data_ptr(), d.data_ptr(), m, n, k, scratch.data_ptr(),
                                     _lib.current_stream_handle()))
    torch.cuda.synchronize()
    return d.cpu().numpy()


@pytest.mark.parametrize("m,n,k", [(128, 32, 32), (300, 32, 576), (1, 64, 64), (257, 64, 800), (4096, 128, 256),
                                   (20000, 128, 96), (513, 256, 2048), (130, 512, 128)])
def test_tc_gemm_matches_float64(m, n, k):
    rs = np.random.RandomState(m + n + k)
    a = rs.randn(m, k).astype(np.float32)
    bt = rs.randn(n, k).astype(np.float32)
    got = _gemm(a, bt)
    ref = a.astype(np.float64) @ bt.astype(np.float64).T
    assert np.isfinite(got).all()
    assert rel_l2(got, ref) < 2e-6


def test_tc_gemm_positive_data_has_no_accumulation_bias():
    """all-positive operands at K=4096: accumulating the whole reduction in the tensor core's truncating fp32 accumulator
    would bias every output low; the chunked accumulation into fp32 registers must not"""
    rs = np.random.RandomState(7)
    a = rs.rand(256, 4096).astype(np.float32)
    bt = rs.rand(128, 4096).astype(np.float32)
    got = _gemm(a, bt)
    ref = a.astype(np.float64) @ bt.astype(np.float64).T
    assert rel_l2(got, ref) < 2e-6
    assert abs(np.mean((got - ref) / ref)) < 2e-6


@pytest.mark.parametrize("m,i,j", [(4096, 128, 128), (5000, 256, 64), (4100, 128, 32), (1031, 384, 256),
                                   (32, 128, 32), (33, 128, 64), (95, 256, 32), (127, 200, 64), (2048, 640, 32),
                                   (3001, 1024, 64), (16384, 128, 64), (777, 136, 96)])
def test_tc_wgrad_matches_float64(m, i, j):
    """The weight-gradient kernel (tc_wgrad.cu) through cpb_debug_tc_wgrad: one / few / many k-blocks per split, ragged
    reduction lengths, I not a multiple of the 128-row tile, and J = 32 / 64 / 96 / 128 / 256 (one or more 32- or 64-wide
    column tiles)."""
    import torch
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(m + i + j)
    big = rs.randn(m, i).astype(np.float32)
    small = rs.randn(m, j).astype(np.float32)
    tb, ts = torch.tensor(big, device="cuda"), torch.tensor(small, device="cuda")
    out = torch.full((i, j), float("nan"), device="cuda")
    part = torch.zeros(2 * i * j, device="cuda")          # the debug entry uses 2 splits
    _lib.check(lib.cpb_debug_tc_wgrad(tb.data_ptr(), ts.data_ptr(), out.data_ptr(), m, i, j, 0, part.data_ptr(),
                                      _lib.current_stream_handle()))
    torch.cuda.synchronize()
    ref = big.astype(np.float64).T @ small.astype(np.float64)
    assert rel_l2(out.cpu().numpy(), ref) < 2e-6


_SNIPPET = r"""
import sys, hashlib, numpy as np, torch
sys.path.insert(0, %r)
from carla_ppo_b200 import _lib
lib = _lib.load()
rs = np.random.RandomState(3)
m, n, k = 3000, 128, 288
a = rs.randn(m, k).astype(np.float32); bt = rs.randn(n, k).astype(np.float32)
ta, tb = torch.tensor(a, device="cuda"), torch.tensor(bt, device="cuda")
d = torch.empty(m, n, device="cuda"); sc = torch.empty(2 * n * k + m * k, device="cuda")
_lib.check(lib.cpb_debug_tc_gemm(ta.data_ptr(), tb.data_ptr(), d.data_ptr(), m, n, k, sc.data_ptr(), _lib.current_stream_handle()))
torch.cuda.synchronize()
print("HASH", hashlib.sha256(d.cpu().numpy().tobytes()).hexdigest())
ref = a.astype(np.float64) @ bt.astype(np.float64).T
print("ERR", float(np.linalg.norm(d.cpu().numpy() - ref) / np.linalg.norm(ref)))
"""


def test_tc_gemm_is_bit_identical_across_cluster_sizes():
    """CPB_TC_CLUSTER only changes who copies which slice of a weight tile (multicast), never the arithmetic."""
    hashes, errs = {}, {}
    for cs in ("1", "2", "4"):
        env = dict(os.environ, CPB_TC_CLUSTER=cs)
        res = subprocess.run([sys.executable, "-c", _SNIPPET % ROOT], env=env, capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stderr[-2000:]
        hashes[cs] = [ln for ln in res.stdout.splitlines() if ln.startswith("HASH")][0]
        errs[cs] = float([ln for ln in res.stdout.splitlines() if ln.startswith("ERR")][0].split()[1])
    assert hashes["1"] == hashes["2"] == hashes["4"]
    assert errs["1"] < 2e-6, errs
