"""The large-batch cases without a GPU: where the live frames of a placed-frame batch sit, and the batches and workspace
sizes of every case of tests/test_large_batch_gpu.py."""
import ctypes as C

import pytest

import large_batch as LB
from harness import lib, library_state, math_mode  # noqa: F401


def base(batch, ct=3, z=64):
    from carla_ppo_b200 import _lib
    return _lib.VaeConfig(batch, ct, z, 0, _lib.FRAME_U8, _lib.FRAME_F32, 1.0 / 255, 1.0, 0.0, 1.0)


def workspace_bytes(lib, case, mode):
    from carla_ppo_b200 import _lib
    with math_mode(lib, mode):
        if "hw" in case:
            return lib.cpb_vae_spec_workspace_bytes(C.byref(_lib.VaeSpec(base(case["batch"]), *case["hw"])), case["ws"])
        spec = _lib.MlpVaeSpec.of(base(case["batch"]), *case["mlp"])
        return lib.cpb_mlpvae_spec_workspace_bytes(C.byref(spec), case["ws"])


def test_live_frames_at_80x160():
    counts = LB.conv_counts(80, 160)
    assert {counts[k] for k in ("xp", "a1", "a2", "a3", "a4")} == {51200, 98592, 43776, 18432, 6144}
    assert LB.live_frames(21781, counts) == [0, 1, 5445, 10485, 10890, 12264, 20971, 21779, 21780]
    assert LB.live_frames(22000, counts) == [0, 1, 5445, 10485, 10890, 12264, 20971, 21781, 21998, 21999]


@pytest.mark.parametrize("name", sorted(LB.CASES))
def test_a_live_frame_on_each_side_of_every_boundary(name):
    case = LB.CASES[name]
    batch = case["batch"]
    live = set(LB.live_frames(batch, LB.counts_of(case)))
    assert {0, 1, batch - 2, batch - 1} <= live
    covered = 0
    for buf, s in LB.counts_of(case).items():
        for k in LB.BOUNDARIES:
            if k < batch * s:                       # the boundary lies inside the buffer
                assert (k - 1) // s in live and k // s in live, (buf, k)
                covered += 1
    assert covered > 0


def test_a_boundary_at_a_frame_start_gets_the_frame_before_it():
    # 512x512: xp holds 2^20 elements per frame, so 2^31 is the first element of frame 2048
    assert LB.conv_counts(512, 512)["xp"] == 1 << 20
    live = LB.live_frames(2100, LB.conv_counts(512, 512))
    assert 2047 in live and 2048 in live


def test_batches_are_the_bounds():
    bound = lambda h, w: ((1 << 31) - 1) // ((h // 2 - 1) * (w // 2 - 1) * 32)
    c = LB.CASES
    assert c["conv80x160-bound"]["batch"] == bound(80, 160) == 21781
    assert c["conv512x512-bound"]["batch"] == bound(512, 512) == 1032
    assert c["conv80x160-simt"]["batch"] * LB.conv_counts(80, 160)["a1"] > 1 << 31
    assert c["conv512x512-simt"]["batch"] * LB.conv_counts(512, 512)["xp"] > 1 << 31
    assert c["conv512x512-simt"]["batch"] * LB.conv_counts(512, 512)["a1"] > 1 << 32
    # the MlpVAE's tensor-core path: batch * 38400 < 2^31
    assert 55924 * 38400 < 1 << 31 <= 55925 * 38400
    assert c["mlp-last-tc"]["batch"] == c["mlp-8192-last-tc"]["batch"] == 55924 and c["mlp-first-fp32"]["batch"] == 55925


@pytest.mark.parametrize("name", sorted(LB.CASES))
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_workspace_bytes(lib, name, mode):
    case = LB.CASES[name]
    assert workspace_bytes(lib, case, mode) == case["bytes"][mode]


def test_only_the_tensor_core_side_plans_mode_2_images():
    """In mode 2 the MlpVAE's workspace at 55 924 frames exceeds the one at 55 925: only a batch on the tensor-core side
    plans the TF32 weight images and split partials; in modes 0 and 1 the workspace grows with the batch."""
    last, first = LB.CASES["mlp-last-tc"], LB.CASES["mlp-first-fp32"]
    assert last["bytes"][2] > first["bytes"][2]
    assert last["bytes"][1] < first["bytes"][1] and last["bytes"][0] < first["bytes"][0]
