"""Host side (CPU) of the on-device policy for any supported SB3 net_arch: the packed layout of every layer (include/quadsim.h,
QsMlpNet), the float64 reference of tests/mlp_ref.py against MlpPolicy.forward_torch, the generalised accuracy criterion,
MlpPolicy.from_sb3, the shapes MlpPolicy refuses, and the qs_rollout_mlp C ABI without a GPU."""
import ctypes as C
import io
import zipfile

import numpy as np
import pytest
import torch

from gym_pybullet_drones_b200 import _native as N
from gym_pybullet_drones_b200.policy import MlpPolicy
from mlp_ref import MlpRef
from qs_testlib import PolicyRef


def _unpack(fr, first):
    """Inverse of MlpPolicy._fragment_order: [Kpad / 16, Npad / 8, 32, 4] int32 -> (hi, lo) float16 [Kpad, Npad]."""
    ksn, ntn = fr.shape[0], fr.shape[1]
    hi = np.zeros((16 * ksn, 8 * ntn), np.uint16)
    lo = np.zeros_like(hi)
    u = fr.numpy().astype(np.int64) & 0xFFFFFFFF
    for lane in range(32):
        g, t = lane // 4, lane % 4
        ka, kb = (4 * t, 4 * t + 2) if first else (2 * t, 2 * t + 8)
        for ks in range(ksn):
            for part, words in ((hi, (0, 1)), (lo, (2, 3))):
                for k, wd in zip((ka, kb), words):
                    v = u[ks, :, lane, wd]
                    part[16 * ks + k, g::8] = v & 0xFFFF
                    part[16 * ks + k + 1, g::8] = v >> 16
    return hi.view(np.float16), lo.view(np.float16)


# (in_dim, out_dim, net_arch): widths that are no multiple of 16 or 64, depth 1 and 4, pi != vf
ARCHS = [(27, 1, [100]), (144, 8, [256, 128, 64, 32]), (57, 6, dict(pi=[128, 64], vf=[256, 256])), (49, 12, [17, 200, 3])]


@pytest.mark.parametrize("in_dim,out_dim,arch", ARCHS)
def test_every_layer_is_packed_as_the_header_defines(in_dim, out_dim, arch):
    """Layer l: [K_l / 16][N_l / 8][32][4] words of the zero-padded hi / lo' parts, K_0 = in_dim padded to 16, hidden widths
    padded to 64, the actor's outputs to 8 nt3 and the critic's to 8; the first layer with the (4t, 4t + 2) k pairs."""
    pol = MlpPolicy.random(in_dim, out_dim, seed=3, critic=True, device="cpu", net_arch=arch, activation="relu")
    for which, net, last in (("actor", pol.actor, 8 * pol.nt3), ("critic", pol.critic, 8)):
        split = pol._split[which]
        assert len(split) == len(net)
        rows = (in_dim + 15) // 16 * 16
        for k, ((w, b), (fr, bp)) in enumerate(zip(net, split)):
            cols = last if k == len(net) - 1 else (w.shape[1] + 63) // 64 * 64
            assert fr.shape == (rows // 16, cols // 8, 32, 4) and fr.dtype == torch.int32 and bp.shape == (cols,)
            wp = np.zeros((rows, cols), np.float32)
            wp[:w.shape[0], :w.shape[1]] = w.numpy()
            hi, lo = _unpack(fr, k == 0)
            want_hi = wp.astype(np.float16)
            want_lo = ((wp - want_hi.astype(np.float32)) * np.float32(2048)).astype(np.float16)
            assert np.array_equal(hi.view(np.uint16), want_hi.view(np.uint16)), (which, k)
            assert np.array_equal(lo.view(np.uint16), want_lo.view(np.uint16)), (which, k)
            assert float(np.abs(bp.numpy()[b.shape[0]:]).max(initial=0.0)) == 0.0 and np.array_equal(bp.numpy()[:b.shape[0]], b.numpy())
            rows = cols


@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_padded_network_evaluates_as_the_unpadded_one(activation):
    """The packed network, unpacked with its padding (hi + lo' / 2048 per weight), evaluates in float64 to the network of the
    unpadded weights' hi + lo' / 2048: padded units are act(0) = 0 and meet zero rows."""
    pol = MlpPolicy.random(49, 12, seed=8, critic=False, device="cpu", net_arch=[17, 200, 3], activation=activation)
    ref = MlpRef(pol)
    padded, plain = [], []
    for k, ((w, _), (fr, bp)) in enumerate(zip(pol.actor, pol._split["actor"])):
        hi, lo = _unpack(fr, k == 0)
        wv = hi.astype(np.float64) + lo.astype(np.float64) / 2048.0
        padded.append((wv, bp.double().numpy()))
        plain.append((wv[:w.shape[0], :w.shape[1]], bp.double().numpy()[:w.shape[1]]))
    x = np.random.default_rng(2).uniform(-2, 2, (33, 49))
    xp = np.zeros((33, padded[0][0].shape[0]))
    xp[:, :49] = x
    yp, y = ref.mlp(padded, xp)[:, :12], ref.mlp(plain, x)
    assert np.abs(yp - y).max() <= 1e-13 * max(1.0, np.abs(y).max())


@pytest.mark.parametrize("in_dim,out_dim,arch", ARCHS + [(72, 4, [64, 64])])
@pytest.mark.parametrize("activation", ["tanh", "relu"])
def test_float64_reference_matches_forward_torch_in_float64(in_dim, out_dim, arch, activation):
    pol = MlpPolicy.random(in_dim, out_dim, seed=in_dim + out_dim, critic=True, log_std=-0.7, device="cpu", net_arch=arch,
                           activation=activation)
    ref = MlpRef(pol)
    g = torch.Generator().manual_seed(3)
    obs = (torch.rand(37, in_dim, generator=g) * 4 - 2).float()
    noise = torch.randn(37, out_dim, generator=g).float()
    raw_t, lp_t, v_t = pol.double().forward_torch(obs.double(), noise.double())
    mean, raw, lp, v = ref.forward(obs, noise)
    assert np.abs(raw - raw_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(raw).max())
    assert np.abs(lp - lp_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(lp).max())
    assert np.abs(v - v_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(v).max())
    raw32, lp32, v32 = pol.forward_torch(obs, noise)         # fp32 itself meets the criterion
    r = ref.check(obs, noise, raw32, lp32, v32)
    assert max(r.values()) <= 1.0, r
    # the other activation is a different network
    assert np.abs(MlpRef(pol, "relu" if activation == "tanh" else "tanh").forward(obs)[0] - ref.forward(obs)[0]).max() > 1e-3


def test_generalised_floor_reproduces_policyref_for_the_default_shape():
    pol = MlpPolicy.random(144, 8, seed=4, critic=True, device="cpu")
    a, b = MlpRef(pol), PolicyRef(pol)
    assert np.array_equal(a.floor_actor, b.floor_actor) and np.array_equal(a.floor_critic, b.floor_critic)


def test_generalised_floor_written_out():
    """Depth 3, Tanh: v0 = 1, v1[k] = 1 + sum_i W1[i,k]^2, v2[k] = 1 + sum_i W2[i,k]^2 v1[i]; ReLU adds no activation term."""
    pol = MlpPolicy.random(10, 2, seed=5, critic=False, device="cpu", net_arch=[5, 4, 3])
    ref = MlpRef(pol)
    w = [l[0] for l in ref.actor]
    v1 = [1 + sum(w[1][i, k] ** 2 for i in range(5)) for k in range(4)]
    v2 = [1 + sum(w[2][i, k] ** 2 * v1[i] for i in range(4)) for k in range(3)]
    for j in range(2):
        want = 6 * 2e-7 * sum(w[3][k, j] ** 2 * v2[k] for k in range(3)) ** 0.5
        assert abs(ref.floor_actor[j] - want) <= 1e-12 * want
    assert float(np.abs(MlpRef(pol, "relu").floor_actor).max()) == 0.0


# ---- from_sb3 (SB3 is not installed here: the key mapping is pinned against a hand-built ActorCriticPolicy state dict) ----
def _sb3_state_dict(in_dim, out_dim, pi, vf, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def seq(prefix, widths):
        for n, (i, o) in enumerate(zip([in_dim] + widths[:-1], widths)):
            sd["%s.%d.weight" % (prefix, 2 * n)] = torch.randn(o, i, generator=g)
            sd["%s.%d.bias" % (prefix, 2 * n)] = torch.randn(o, generator=g)
    seq("mlp_extractor.policy_net", pi)
    seq("mlp_extractor.value_net", vf)
    sd["action_net.weight"], sd["action_net.bias"] = torch.randn(out_dim, pi[-1], generator=g), torch.randn(out_dim, generator=g)
    sd["value_net.weight"], sd["value_net.bias"] = torch.randn(1, vf[-1], generator=g), torch.randn(1, generator=g)
    sd["log_std"] = torch.randn(out_dim, generator=g)
    return sd


def test_from_sb3_state_dict_and_zip(tmp_path):
    sd = _sb3_state_dict(27, 4, [128, 64, 32, 16], [256], seed=1)
    lin = lambda pre, n: [torch.nn.Linear(1, 1) for _ in range(n)]   # noqa: E731
    pi, vf = lin("pi", 5), lin("vf", 2)
    for mods, keys in ((pi, ["mlp_extractor.policy_net.%d" % i for i in (0, 2, 4, 6)] + ["action_net"]),
                       (vf, ["mlp_extractor.value_net.0", "value_net"])):
        for m, k in zip(mods, keys):
            m.weight, m.bias = torch.nn.Parameter(sd[k + ".weight"]), torch.nn.Parameter(sd[k + ".bias"])
    want = MlpPolicy.from_linear(pi, sd["log_std"], vf, device="cpu", activation="relu")
    path = tmp_path / "best_model.zip"
    buf = io.BytesIO()
    torch.save(sd, buf)
    with zipfile.ZipFile(path, "w") as z:
        z.writestr("data", "{}")
        z.writestr("policy.pth", buf.getvalue())
    x = torch.randn(9, 27, generator=torch.Generator().manual_seed(2))
    for src in (sd, str(path), path):
        got = MlpPolicy.from_sb3(src, activation="relu", device="cpu")
        assert got.net_arch == dict(pi=[128, 64, 32, 16], vf=[256]) and got.activation == "relu" and not got.classic
        for a, b in zip(got.forward_torch(x), want.forward_torch(x)):
            assert torch.equal(a, b)
    assert MlpPolicy.from_sb3(_sb3_state_dict(144, 8, [64, 64], [64, 64], 3), device="cpu").classic


@pytest.mark.parametrize("key", ["mlp_extractor.shared_net.0.weight", "features_extractor.linear.weight", "action_dist.log_std",
                                 "mlp_extractor.policy_net.0.scale"])
def test_from_sb3_refuses_parameters_outside_the_mapping(key):
    sd = _sb3_state_dict(27, 4, [64, 64], [64, 64], seed=2)
    sd[key] = torch.zeros(3)
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        MlpPolicy.from_sb3(sd, device="cpu")


def test_from_sb3_refuses_an_incomplete_policy():
    sd = _sb3_state_dict(27, 4, [64, 64], [64, 64], seed=2)
    del sd["log_std"]
    with pytest.raises(ValueError, match="log_std"):
        MlpPolicy.from_sb3(sd, device="cpu")


# ---- refusals --------------------------------------------------------------------------------------------------------
def _net(dims, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(i, o, generator=g), torch.randn(o, generator=g)) for i, o in zip(dims[:-1], dims[1:])]


@pytest.mark.parametrize("actor,critic,activation,match", [
    (_net([20, 4]), None, "tanh", "0 hidden layers"),
    (_net([20, 8, 8, 8, 8, 8, 4]), None, "tanh", "5 hidden layers"),
    (_net([20, 257, 4]), None, "tanh", "257 units wide"),
    (_net([20, 64, 4]), _net([20, 300, 1]), "tanh", "300 units wide"),
    (_net([20, 64, 4]), None, "sigmoid", "activation"),
    (_net([20, 64, 33]), None, "tanh", "32 action outputs"),
    (_net([20, 64, 4]), _net([21, 64, 1]), "relu", "critic input width"),
])
def test_out_of_scope_shapes_are_refused(actor, critic, activation, match):
    with pytest.raises(ValueError, match=match) as ei:
        MlpPolicy(actor, torch.zeros(actor[-1][0].shape[1]), critic, device="cpu", activation=activation)
    if "layers" in match or "wide" in match or "activation" in match:
        assert "forward_torch + step()" in str(ei.value) and "256" in str(ei.value)


def test_random_net_arch_forms_and_default_unchanged():
    a = MlpPolicy.random(30, 4, seed=9, device="cpu")
    b = MlpPolicy.random(30, 4, seed=9, device="cpu", net_arch=[64, 64], activation="tanh")
    assert a.classic and a.net_arch == dict(pi=[64, 64], vf=[64, 64]) and a.HIDDEN == 64 and a.nt3 == 1
    for (wa, ba), (wb, bb) in zip(a.actor + a.critic, b.actor + b.critic):
        assert torch.equal(wa, wb) and torch.equal(ba, bb)
    c = MlpPolicy.random(30, 4, seed=9, device="cpu", net_arch=dict(pi=[32], vf=[128, 128, 8]))
    assert c.net_arch == dict(pi=[32], vf=[128, 128, 8]) and not c.classic and c.max_width == 128
    with pytest.raises(ValueError, match="QsPolicy"):
        c.c_struct()


# ---- C ABI (no GPU) -----------------------------------------------------------------------------------------------------
def test_mlp_abi_exports_and_struct_layout():
    lib = N.lib()
    for s in ("qs_rollout_mlp", "qs_rollout_mlp_max_ticks", "qs_sizeof_mlp_policy"):
        assert s in N.EXPORTS and getattr(lib, s) is not None
    assert lib.qs_sizeof_mlp_policy() == C.sizeof(N.QsMlpPolicy)
    assert C.sizeof(N.QsMlpNet) == 10 * 8 + 6 * 4
    assert lib.qs_rollout_mlp_max_ticks(N.ACT_RPM, 15, 2, 0) == 0 and lib.qs_rollout_mlp_max_ticks(N.ACT_RPM, 15, 2, 257) == 0
    assert lib.qs_rollout_mlp_max_ticks(N.ACT_RPM, 15, 65, 64) == 0
    t64, t256 = lib.qs_rollout_mlp_max_ticks(N.ACT_RPM, 15, 2, 64), lib.qs_rollout_mlp_max_ticks(N.ACT_RPM, 15, 2, 256)
    assert 0 < t256 <= t64 <= lib.qs_rollout_max_ticks(N.ACT_RPM, 15, 2), (t64, t256)


def _mlp_call(lib, mutate, act_type=N.ACT_RPM, D=2, effects=0, T=4, rio_policy=False):
    buf = (C.c_char * 8192)()
    base = (C.addressof(buf) + 63) & ~63
    P, st, rio, q = N.QsParams(), N.QsState(), N.QsRolloutIO(), N.QsMlpPolicy()
    st.planes, st.step_counter, st.target_pos, st.pid, st.last_rpm = base, base + 2048, base + 1024, base + 3072, base + 4096
    rio.obs_init, rio.obs, rio.reward, rio.terminated, rio.truncated = base + 512, base + 768, base + 1280, base + 1536, base + 1600
    rio.T, rio.act_buffer_size = T, 15
    A = {N.ACT_RPM: 4, N.ACT_PID: 3, N.ACT_ONE_D_RPM: 1}[act_type]
    for net, depth, tiles in ((q.actor, 2, 1), (q.critic, 2, 1)):
        net.depth, net.out_tiles = depth, tiles
        for l in range(depth + 1):
            net.w[l], net.b[l] = base, base
        for l in range(depth):
            net.width[l] = 256
    q.in_dim, q.out_dim, q.log_std = D * (12 + 15 * A), D * A, base
    mutate(q)
    if rio_policy:
        rio.policy = base
    rc = lib.qs_rollout_mlp(C.byref(P), C.byref(st), C.byref(rio), C.byref(q), act_type, 1, 4, D, 8, effects, 0, None)
    return rc, lib.qs_last_error().decode()


def _set(field, value, net="actor"):
    def f(q):
        obj = getattr(q, net)
        if isinstance(field, tuple):
            getattr(obj, field[0])[field[1]] = value
        else:
            setattr(obj, field, value) if hasattr(obj, field) else setattr(q, field, value)
    return f


@pytest.mark.parametrize("mutate,kw,code,match", [
    (_set("depth", 0), {}, -3, "hidden layers"),
    (_set("depth", 5), {}, -3, "hidden layers"),
    (_set(("width", 1), 320), {}, -3, "multiples of 64 up to 256"),
    (_set(("width", 0), 96, "critic"), {}, -3, "critic"),
    (_set("out_tiles", 3), {}, -3, "out_tiles"),
    (_set("out_tiles", 2, "critic"), {}, -3, "out_tiles"),
    (lambda q: setattr(q, "activation", 7), {}, -4, "activation"),
    (_set(("w", 2), None), {}, -1, "layer 2 weights are NULL"),
    (_set(("w", 1), 8200), {}, -2, "aligned"),
    (lambda q: setattr(q, "out_dim", 7), {}, -3, "in_dim/out_dim"),
    (lambda q: setattr(q, "log_std", None), {}, -1, "log_std"),
    (lambda q: (setattr(q.critic, "depth", 0), setattr(q, "values", 64)), {}, -1, "without a critic"),
    (lambda q: None, {"T": 5000}, -5, "max_ticks"),
    (lambda q: None, {"effects": 5}, -5, "GND|DW"),
    (lambda q: None, {"rio_policy": True}, -5, "QsRolloutIO.policy must be NULL"),
])
def test_mlp_entry_argument_errors_without_a_gpu(mutate, kw, code, match):
    rc, msg = _mlp_call(N.lib(), mutate, **kw)
    assert rc == code and match in msg and msg.startswith("qs_rollout_mlp: "), (rc, msg)


def test_mlp_entry_null_policy_and_drones_per_env():
    lib = N.lib()
    assert lib.qs_rollout_mlp(None, None, None, None, 0, 1, 4, 2, 8, 0, 0, None) == -1
    rc, msg = _mlp_call(lib, lambda q: setattr(q, "in_dim", 65 * 27) or setattr(q, "out_dim", 65), act_type=N.ACT_ONE_D_RPM, D=65)
    assert rc == -5 and "drones_per_env <= 64" in msg and msg.startswith("qs_rollout_mlp: "), (rc, msg)
