"""PPO policy / value trunks of any depth without a GPU: the float64 restatement (tests/ppo_restatement.py) against
oracle/ppo_oracle.py bit for bit at two layers per trunk and against torch autograd elsewhere; cpb_ppo_spec layouts,
names and workspace sizes; the refusals of a bad spec; the checkpoint architecture reader and the train.py flags."""
import ctypes as C

import numpy as np
import pytest

import ppo_restatement as pr
from harness import lib, library_state  # noqa: F401
from oracle import ppo_oracle as po
from ppo_cases import bounds
from ppo_checks import ppo_call, SPEC_ENTRIES, torch_loss_and_grads

ARCHS = [((1,), (1,)), ((3, 2), (1,)), ((7,), (4, 4, 4)), ((64,), (64,)), ((256, 256), (256, 256, 256)),
         ((33, 7, 65), (31,)), ((64,) * 8, (32,) * 8), ((2048,), (1024, 1024)), ((500, 300), (500, 300))]


def _batch(S, A, n, seed):
    rs = np.random.RandomState(seed)
    low, high = bounds(A)
    s = rs.randn(n, S)
    a = np.clip(rs.randn(n, A) * 0.3 + (low + high) / 2, low, high)
    return s, a, rs.randn(n) + 1.0, rs.randn(n), low, high


def _perturbed(p, seed, scale=0.05):
    rs = np.random.RandomState(seed)
    return {k: (v + scale * rs.randn(*v.shape)).astype(np.float64) for k, v in p.items()}


def test_oracle_equals_ppo_oracle_bit_for_bit_at_two_layers():
    S, A, H = 20, 2, (12, 9)
    p = {k: v.astype(np.float64) for k, v in pr.init_params(S, bounds(A), H, H, seed=1).items()}
    p = _perturbed(p, 2)
    old = _perturbed(p, 3, 0.02)
    s, a, ret, adv, low, high = _batch(S, A, 37, 4)
    mine = pr.loss_and_grads(p, old, s, a, ret, adv, (low, high), 0.2, 1.0, 0.01)
    ref = po.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    for k in ("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio"):
        assert mine[k] == ref[k], k
    assert set(mine["grads"]) == set(ref["grads"]) == set(po.PPO_TENSORS)
    for k in po.PPO_TENSORS:
        assert np.array_equal(mine["grads"][k], ref["grads"][k]), k
    assert all(np.array_equal(x, y) for x, y in zip(pr.forward(p, s, (low, high)), po.forward(p, s, low, high)))
    # learn: Adam over 2 epochs x 3 minibatches, records and parameters
    from oracle.vae_oracle import adam_init_state
    T = 40
    rs = np.random.RandomState(5)
    states, actions = rs.randn(T, S), np.clip(rs.randn(T, A) * 0.3, low, high)
    vals, rews, dones = rs.randn(T), rs.randn(T), (rs.rand(T) < 0.1).astype(np.float64)
    perms = [rs.permutation(T) for _ in range(2)]
    pa, pb = {k: v.copy() for k, v in p.items()}, {k: v.copy() for k, v in p.items()}
    sa, sb = adam_init_state(pa), adam_init_state(pb)
    rec_ref = po.learn(pa, sa, states, actions, vals, rews, dones, 0.3, low, high, num_epochs=2, batch_size=16, perms=perms)
    rec, applied = pr.learn(pb, sb, states, actions, vals, rews, dones, 0.3, (low, high), num_epochs=2, batch_size=16,
                            perms=perms)
    assert applied == len(rec_ref)
    assert np.array_equal(np.asarray(rec_ref, np.float64), rec[:, :5])
    for k in pa:
        assert np.array_equal(pa[k], pb[k]), k


@pytest.mark.parametrize("arch", [((1,), (1,)), ((3, 2), (1,)), ((7,), (4, 4, 4))])
def test_oracle_matches_torch_autograd(arch):
    pytest.importorskip("torch")
    pol, val = arch
    S, A = 5, 3
    p = _perturbed({k: v.astype(np.float64) for k, v in pr.init_params(S, bounds(A), pol, val, seed=7).items()}, 8, 0.3)
    old = _perturbed(p, 9, 0.05)
    s, a, ret, adv, low, high = _batch(S, A, 23, 10)
    ref = pr.loss_and_grads(p, old, s, a, ret, adv, (low, high), 0.2, 1.0, 0.01)
    loss, grads = torch_loss_and_grads(p, old, s, a, ret, adv, (low, high), 0.2, 1.0, 0.01)
    assert abs(loss - ref["loss"]) <= 1e-10
    for k, g in grads.items():
        assert np.max(np.abs(g - ref["grads"][k])) <= 1e-10, k


def test_options_rule_runs_on_top_of_the_oracle():
    """The clipping / KL rule of the restatement on a non-default network: a clip that binds and a stop."""
    S, A, pol, val = 6, 2, (9, 5, 3), (4,)
    p = _perturbed({k: v.astype(np.float64) for k, v in pr.init_params(S, bounds(A), pol, val, seed=11).items()}, 12, 0.2)
    rs = np.random.RandomState(13)
    T = 64
    low, high = bounds(A)
    states, actions = rs.randn(T, S), np.clip(rs.randn(T, A) * 0.3, low, high)
    vals, rews, dones = rs.randn(T), rs.randn(T), np.zeros(T)
    perms = [rs.permutation(T) for _ in range(3)]
    from oracle.vae_oracle import adam_init_state
    rec, applied = pr.learn({k: v.copy() for k, v in p.items()}, adam_init_state(p), states, actions, vals, rews, dones, 0.3,
                            (low, high), lr=3e-2, num_epochs=3, batch_size=16, perms=perms, max_grad_norm=1e-3, target_kl=1e-4)
    assert 1 <= applied < len(rec)
    assert np.isnan(rec[applied + 1:]).all() and np.isfinite(rec[:applied + 1]).all()
    assert (rec[:applied + 1, 6] > 1e-3).all()          # every evaluated gradient was clipped


def _spec(lib_mod, S, A, pol, val, h1=0, h2=0):
    cfg = lib_mod.PpoConfig()
    cfg.state_dim, cfg.num_actions = S, A
    sp = lib_mod.PpoSpec.of(cfg, pol, val)
    sp.base.hidden1, sp.base.hidden2 = h1, h2
    return sp


@pytest.mark.parametrize("arch", ARCHS)
def test_spec_layout_and_names_match_the_oracle(lib, arch):
    from carla_ppo_b200 import _lib
    pol, val = arch
    S, A = 67, 2
    sp = _spec(_lib, S, A, pol, val)
    n = lib.cpb_ppo_spec_num_tensors(C.byref(sp))
    ref = pr.param_shapes(S, bounds(A), pol, val)
    assert n == len(ref) == 2 * (len(pol) + len(val)) + 5
    names = [lib.cpb_ppo_spec_tensor_name(C.byref(sp), i).decode() for i in range(n)]
    assert names == list(ref)
    assert lib.cpb_ppo_spec_tensor_name(C.byref(sp), n) is None
    offs, sizes, shapes, total = (C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int32 * (2 * n))(), C.c_int64()
    assert lib.cpb_ppo_spec_layout(C.byref(sp), offs, sizes, shapes, C.byref(total)) == 0
    end = 0
    for i, (name, shape) in enumerate(ref.items()):
        got = tuple(v for v in shapes[2 * i:2 * i + 2] if v > 0)
        assert got == shape, name
        assert sizes[i] == int(np.prod(shape))
        assert offs[i] % 64 == 0 and offs[i] >= end, name
        end = offs[i] + sizes[i]
    assert total.value >= end and total.value % 64 == 0
    assert pr.architecture(pr.init_params(S, bounds(A), pol, val)) == (tuple(pol), tuple(val))


@pytest.mark.parametrize("hidden", [(500, 300), (17, 5)])
def test_legacy_equals_twin_at_two_layers(lib, hidden):
    from carla_ppo_b200 import _lib
    h1, h2 = hidden
    cfg = _lib.PpoConfig()
    cfg.state_dim, cfg.num_actions, cfg.hidden1, cfg.hidden2 = 67, 2, h1, h2
    sp = _lib.PpoSpec.of(cfg, hidden, hidden)
    n = lib.cpb_ppo_num_tensors()
    assert n == lib.cpb_ppo_spec_num_tensors(C.byref(sp)) == 13
    assert [lib.cpb_ppo_tensor_name(i) for i in range(n)] == [lib.cpb_ppo_spec_tensor_name(C.byref(sp), i) for i in range(n)]
    a = [(C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int32 * (2 * n))(), C.c_int64()]
    b = [(C.c_int64 * n)(), (C.c_int64 * n)(), (C.c_int32 * (2 * n))(), C.c_int64()]
    assert lib.cpb_ppo_layout(C.byref(cfg), a[0], a[1], a[2], C.byref(a[3])) == 0
    assert lib.cpb_ppo_spec_layout(C.byref(sp), b[0], b[1], b[2], C.byref(b[3])) == 0
    assert [list(x) for x in a[:3]] == [list(x) for x in b[:3]] and a[3].value == b[3].value
    for mb, hz in ((1, 0), (256, 0), (64, 2048), (8200, 8200)):
        assert lib.cpb_ppo_workspace_bytes(C.byref(cfg), mb, hz) == lib.cpb_ppo_spec_workspace_bytes(C.byref(sp), mb, hz) > 0


def _bad_specs():
    from carla_ppo_b200 import _lib
    good = ((64, 64), (32,))
    out = {"depth0_policy": _spec(_lib, 67, 2, *good), "depth9_value": _spec(_lib, 67, 2, *good),
           "width0": _spec(_lib, 67, 2, (64, 0), (32,)), "width_neg": _spec(_lib, 67, 2, (64,), (-3,)),
           "hidden1": _spec(_lib, 67, 2, *good, h1=500), "hidden2": _spec(_lib, 67, 2, *good, h2=300),
           "actions0": _spec(_lib, 67, 0, *good), "actions5": _spec(_lib, 67, 5, *good),
           "state0": _spec(_lib, 0, 2, *good)}
    out["depth0_policy"].num_policy = 0
    out["depth9_value"].num_value = 9
    return out


@pytest.mark.parametrize("bad", list(_bad_specs()) + ["null"])
def test_bad_specs_are_refused_before_any_launch(lib, bad):
    sp = None if bad == "null" else C.byref(_bad_specs()[bad])
    before = lib.cpb_launch_count()
    for entry in SPEC_ENTRIES:
        assert ppo_call(lib, "cpb_ppo_spec_", entry, sp) == -1, entry          # CPB_ERR_INVALID_ARGUMENT
    assert lib.cpb_ppo_spec_tensor_name(sp, 0) is None
    assert lib.cpb_launch_count() == before


def _blob(S, pol, val, record=True):
    from carla_ppo_b200.ppo import ARCH_KEYS
    blob = {"policy/" + k: v for k, v in pr.init_params(S, bounds(2), pol, val).items()}
    if record:
        blob[ARCH_KEYS[0]], blob[ARCH_KEYS[1]] = np.asarray(pol, np.int32), np.asarray(val, np.int32)
    return blob


def test_blob_architecture_reader():
    from carla_ppo_b200.ppo import blob_architecture
    for pol, val in ARCHS:
        for record in (True, False):
            assert blob_architecture(_blob(67, pol, val, record)) == (tuple(pol), tuple(val))
    with pytest.raises(ValueError):
        blob_architecture({"policy/dense/kernel": np.zeros((3, 4))})


def test_a_width_equal_to_the_state_size_is_never_guessed(tmp_path):
    """state_dim 64 (z_dim 61 + 3 measurements) and (64, 64) / (64, 64): the dense kernels alone also fit (64) / (64, 64,
    64) and (64, 64, 64) / (64).  The recorded architecture settles it; without the record the checkpoint is refused
    (blob_architecture, checkpoint_architecture, and so load_blob and a resumed train.py run), never guessed."""
    from carla_ppo_b200.ppo import ARCH_KEYS, blob_architecture, checkpoint_architecture
    pol = val = (64, 64)
    assert blob_architecture(_blob(64, pol, val)) == (pol, val)
    assert blob_architecture(_blob(64, (64,), (64, 64, 64))) == ((64,), (64, 64, 64))
    with pytest.raises(ValueError, match=r"several architectures .*policy \[64, 64\] / value \[64, 64\]"):
        blob_architecture(_blob(64, pol, val, record=False))
    wrong = _blob(64, pol, val)
    wrong[ARCH_KEYS[1]] = np.asarray((64, 64, 64), np.int32)        # a record that the variables do not have
    with pytest.raises(ValueError, match="which its variables do not have"):
        blob_architecture(wrong)
    for record, expect in ((True, (pol, val)), (False, None)):
        d = tmp_path / str(record)
        d.mkdir()
        np.savez(str(d / "model.ckpt-1.npz"), **_blob(64, pol, val, record))
        (d / "checkpoint").write_text('model_checkpoint_path: "model.ckpt-1"\n')
        if expect is None:
            with pytest.raises(ValueError, match="several architectures"):
                checkpoint_architecture(str(d))
        else:
            assert checkpoint_architecture(str(d)) == expect
    assert checkpoint_architecture(str(tmp_path / "none")) is None


def test_train_flags_and_checkpoint_architecture():
    from carla_ppo_b200.train import resolve_architecture
    d = (500, 300)
    assert resolve_architecture(None, None, None) == (d, d)
    assert resolve_architecture([256, 256], None, None) == ((256, 256), d)
    ck = ((256, 256), (256, 256, 256))
    assert resolve_architecture(None, None, ck) == ck
    assert resolve_architecture([256, 256], [256, 256, 256], ck) == ck
    with pytest.raises(ValueError, match="--value_hidden_sizes 500 300 disagrees"):
        resolve_architecture(None, [500, 300], ck)
