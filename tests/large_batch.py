"""The large-batch cases of tests/test_large_batch_gpu.py and the rule that places their live frames (pinned without a
GPU by tests/test_large_batch_cpu.py).

A placed-frame batch is almost all null frames -- source 0, target 0.5, eps 0, every bias 0, MSE loss -- each of which
computes exactly 0 in every buffer and contributes exactly 0 to every gradient, in all three math modes.  Its live
frames sit where 32-bit element offsets break: for every checked buffer with s elements per frame and every
k = 2^29 .. 2^32 inside the buffer, the frames that hold elements k - 1 and k (one frame when it straddles k), plus
frames 0, 1, B - 2 and B - 1."""
BOUNDARIES = [1 << 29, 1 << 30, 1 << 31, 1 << 32]


def sides(h, w):
    out = [(h, w)]
    for _ in range(4):
        h, w = (h - 4) // 2 + 1, (w - 4) // 2 + 1
        out.append((h, w))
    return out


def conv_counts(h, w):
    """Elements per frame of every [B, ...] buffer of the ConvVAE at h x w (xp and logits_p hold 4 channels)."""
    s = sides(h, w)
    area = lambda lv: s[lv][0] * s[lv][1]
    return {"xp": area(0) * 4, "logits_p": area(0) * 4, "a1": area(1) * 32, "b3": area(1) * 32, "gA": area(1) * 32,
            "gB": area(1) * 32, "a2": area(2) * 64, "b2": area(2) * 64, "a3": area(3) * 128, "b1": area(3) * 128,
            "a4": area(4) * 256, "d1": area(4) * 256}


def mlp_counts(enc, dec, ct=3):
    """Elements per frame of every [B, width] buffer of the MlpVAE."""
    out = {"x": 38400, "logits": 12800 * ct}
    out.update({"h%d" % i: v for i, v in enumerate(enc)})
    out.update({"g%d" % j: v for j, v in enumerate(dec)})
    return out


def live_frames(batch, counts):
    live = {0, 1, batch - 2, batch - 1}
    for s in set(counts.values()):
        for k in BOUNDARIES:
            for e in (k - 1, k):
                if e // s < batch:
                    live.add(e // s)
    return sorted(f for f in live if f >= 0)


# One entry per case: the model, the batch, the math modes, the calls, the largest workspace the case allocates
# (cpb_*_spec_workspace_bytes of that call kind per mode: the ConvVAE's does not depend on the mode, the MlpVAE's grows
# in mode 2 by the TF32 weight images and k-split partials of the tensor-core path).
WS_ENCODE, WS_FORWARD, WS_TRAIN = 0, 1, 2
CASES = {
    "conv80x160-bound": dict(hw=(80, 160), batch=21781, modes=(1, 2), ws=WS_TRAIN, bytes={m: 59903188224 for m in (0, 1, 2)}),
    "conv80x160-simt": dict(hw=(80, 160), batch=22000, modes=(0,), ws=WS_TRAIN, bytes={m: 60504541184 for m in (0, 1, 2)}),
    "conv512x512-bound": dict(hw=(512, 512), batch=1032, modes=(1, 2), ws=WS_FORWARD, bytes={m: 44727743232 for m in (0, 1, 2)}),
    "conv512x512-simt": dict(hw=(512, 512), batch=2100, modes=(0,), ws=WS_ENCODE, bytes={m: 41104839168 for m in (0, 1, 2)}),
    "mlp-last-tc": dict(mlp=((512, 256), (256, 512)), batch=55924, modes=(2,), ws=WS_TRAIN,
                        bytes={0: 26980972032, 1: 26980972032, 2: 27910960640}),
    "mlp-first-fp32": dict(mlp=((512, 256), (256, 512)), batch=55925, modes=(0, 1, 2), ws=WS_TRAIN,
                           bytes={m: 26981448704 for m in (0, 1, 2)}),
    "mlp-8192-last-tc": dict(mlp=((8192,), (8192,)), batch=55924, modes=(2,), ws=WS_TRAIN,
                             bytes={0: 36135163392, 1: 36135163392, 2: 51014981120}),
}


def counts_of(case):
    return conv_counts(*case["hw"]) if "hw" in case else mlp_counts(*case["mlp"])
