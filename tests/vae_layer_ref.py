"""Torch restatement of the ConvVAE's three convolution contractions, for the per-layer GPU tests.

The same im2col + matmul formulation as oracle/vae_oracle.py's conv_gather / conv_scatter / conv_wgrad (pinned to them
by tests/test_vae_layers_cpu.py), written for torch tensors so that the per-layer tests can evaluate it on the GPU in
float64 (the reference) and in float32 with TF32 off (the error yardstick) on the device's own operands.  Notation as
in the oracle: a stride-2 layer connects a "big" image [B,Hb,Wb,Cb] and a "small" image [B,Hs,Ws,Cs] through a kernel
[k,k,Cb,Cs]."""
import torch


def _windows(big, k, hs, ws):
    """[B,Hb,Wb,Cb] -> [B*hs*ws, k*k*Cb]: the stride-2 windows big[b, 2i+kh, 2j+kw, c] as rows (im2col)."""
    big = big.contiguous()
    b, _, _, cb = big.shape
    sb, sh, sw, sc = big.stride()
    return big.as_strided((b, hs, ws, k, k, cb), (sb, 2 * sh, 2 * sw, sh, sw, sc)).reshape(b * hs * ws, k * k * cb)


def gather(big, w):
    """small[b,i,j,cs] = sum_{kh,kw,cb} big[b,2i+kh,2j+kw,cb] * w[kh,kw,cb,cs]  (vae_oracle.conv_gather)."""
    k = w.shape[0]
    b, hb, wb, cb = big.shape
    hs, ws = (hb - k) // 2 + 1, (wb - k) // 2 + 1
    return (_windows(big, k, hs, ws) @ w.reshape(k * k * cb, -1)).reshape(b, hs, ws, -1)


def scatter(small, w, out_hw):
    """big[b,2i+kh,2j+kw,cb] += small[b,i,j,cs] * w[kh,kw,cb,cs] into a [B, out_hw, Cb] image of zeros
    (vae_oracle.conv_scatter with out_hw)."""
    k = w.shape[0]
    b, hs, ws, cs = small.shape
    big = small.new_zeros((b, out_hw[0], out_hw[1], w.shape[2]))
    flat = small.reshape(-1, cs)
    for kh in range(k):
        for kw in range(k):
            big[:, kh:kh + 2 * hs:2, kw:kw + 2 * ws:2, :] += (flat @ w[kh, kw].T).reshape(b, hs, ws, -1)
    return big


def wgrad(big, small, k):
    """gw[kh,kw,cb,cs] = sum_{b,i,j} big[b,2i+kh,2j+kw,cb] * small[b,i,j,cs]  (vae_oracle.conv_wgrad)."""
    b, hs, ws, cs = small.shape
    cb = big.shape[3]
    return (_windows(big, k, hs, ws).T @ small.reshape(-1, cs)).reshape(k, k, cb, cs)


def heads_dgrad(gheads, wm, wl):
    """d loss / d flat(a4) = gmean Wm^T + glogvar Wl^T from the library's [2, B, z_pad] gradient rows: the first z
    columns, z = the kernels' width (the padded columns meet zero rows of the library's padded kernels)."""
    z = wm.shape[1]
    return gheads[0][:, :z] @ wm.T + gheads[1][:, :z] @ wl.T


def dense1_fwd(latent, wd):
    """dense1 without its bias from the library's [B, z_pad] latent rows: their first z columns times the [z, 6144]
    kernel."""
    return latent[:, :wd.shape[0]] @ wd


def round_tf32(t):
    """float32 tensor -> the nearest TF32 values (ties away from zero: bits + 0x1000, then the 13 low bits cleared), as
    float32: tests/tf32_oracle.round_tf32 for torch tensors."""
    bits = t.to(torch.float32).contiguous().view(torch.int32)
    return ((bits + 0x1000) & -0x2000).view(torch.float32)
