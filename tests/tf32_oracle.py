"""The "TF32 restatement" of the float64 oracle (test infrastructure for math mode 2).

Math mode 2 multiplies the operands of the tensor-core contractions -- forward, data gradient and weight gradient of
conv2-4 and deconv1-3 -- after rounding both to the nearest TF32 value, and sums in fp32.  The restatement is
oracle.vae_oracle with exactly those operands rounded, everything else in float64; it plays the role for mode 2 that
the float32 CPU restatement plays for mode 1.

It reuses the oracle unchanged: while a restatement runs, the oracle module's three convolution primitives are
replaced by versions that round their operands when the contraction belongs to a tensor-core layer.  A contraction
is one of the edge layers (conv1, deconv4: fp32 kernels in every mode) exactly when its big image has the 3 channels
of the source frame or the 1 / 3 channels of the target; every tensor-core layer's big image has 32, 64 or 128.  The
dense layers use `@` directly and are never rounded."""
import contextlib

import numpy as np

from oracle import vae_oracle as vo

EDGE_CHANNELS = (1, 3)


def round_tf32(a):
    """a rounded to float32, then to the nearest TF32 value (10-bit mantissa, ties away from zero: bits + 0x1000, then
    the 13 low bits cleared) -- the operand rounding of math mode 2.  Returns float64."""
    bits = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((bits + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32).astype(np.float64)


@contextlib.contextmanager
def rounded_tensor_core_contractions(tc_round=round_tf32):
    """Within the block, the oracle's conv_gather / conv_scatter / conv_wgrad apply tc_round to both operands of every
    tensor-core layer's contraction.  Counts the rounded and the plain calls in the yielded dict."""
    gather, scatter, wgrad = vo.conv_gather, vo.conv_scatter, vo.conv_wgrad
    calls = {"rounded": 0, "plain": 0}

    def tc(cb):
        hit = cb not in EDGE_CHANNELS
        calls["rounded" if hit else "plain"] += 1
        return hit

    def conv_gather(big, w):
        return gather(tc_round(big), tc_round(w)) if tc(w.shape[2]) else gather(big, w)

    def conv_scatter(small, w, out_hw=None):
        return scatter(tc_round(small), tc_round(w), out_hw) if tc(w.shape[2]) else scatter(small, w, out_hw)

    def conv_wgrad(big, small, k):
        return wgrad(tc_round(big), tc_round(small), k) if tc(big.shape[3]) else wgrad(big, small, k)

    vo.conv_gather, vo.conv_scatter, vo.conv_wgrad = conv_gather, conv_scatter, conv_wgrad
    try:
        yield calls
    finally:
        vo.conv_gather, vo.conv_scatter, vo.conv_wgrad = gather, scatter, wgrad


def loss_and_grads(params, x, y, eps, loss_type="mse", tc_round=round_tf32, **kw):
    """vae_oracle.loss_and_grads with tc_round applied to both operands of the tensor-core contractions."""
    with rounded_tensor_core_contractions(tc_round):
        return vo.loss_and_grads(params, x, y, eps, loss_type, **kw)
