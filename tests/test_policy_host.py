"""Host side of the on-device policy (CPU): the fragment-ordered weight layout of include/quadsim.h (QsPolicy) and the two-term
float16 split it stores."""
import numpy as np
import pytest
import torch

from gym_pybullet_drones_b200.policy import MlpPolicy
from qs_testlib import PolicyRef


def _words(part):
    return part.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF


def test_fragment_order_matches_the_header_definition():
    torch.manual_seed(0)
    K, Nc = 48, 16
    hi, lo = torch.randn(K, Nc).to(torch.float16), torch.randn(K, Nc).to(torch.float16)
    for first in (False, True):
        fr = MlpPolicy._fragment_order(hi, lo, first)
        assert fr.shape == (K // 16, Nc // 8, 32, 4) and fr.dtype == torch.int32
        for ks in range(K // 16):
            for n in range(Nc // 8):
                for lane in range(32):
                    g, t = lane // 4, lane % 4
                    ka, kb = (4 * t, 4 * t + 2) if first else (2 * t, 2 * t + 8)
                    for w, (part, k) in enumerate(((hi, ka), (hi, kb), (lo, ka), (lo, kb))):
                        u = _words(part)
                        want = int(u[16 * ks + k, 8 * n + g]) | (int(u[16 * ks + k + 1, 8 * n + g]) << 16)
                        assert (int(fr[ks, n, lane, w]) & 0xFFFFFFFF) == want, (first, ks, n, lane, w)


def test_two_term_split_reproduces_fp32_weights():
    """hi + lo' / 2048 equals the fp32 weight to ~2^-22 relative -- below the fp16 normal range (|w| < 6e-5) to 2e-11 absolute --
    which is what makes the tensor-core product fp32-accurate."""
    g = torch.Generator().manual_seed(1)
    w = (torch.rand(144, 64, generator=g) * 2 - 1) * torch.logspace(-4, 1, 64)
    hi = w.to(torch.float16)
    lo = ((w - hi.to(torch.float32)) * 2048.0).to(torch.float16)
    back = hi.to(torch.float64) + lo.to(torch.float64) / 2048.0
    err = (back - w.to(torch.float64)).abs()
    assert bool((err <= 2.0 ** -21 * w.abs().to(torch.float64) + 2e-11).all())


def test_prepare_pads_rows_to_16_and_last_columns_to_8():
    pol = MlpPolicy.random(27, 1, seed=2, critic=True, device="cpu")        # HoverAviary ONE_D_RPM: in 27, out 1
    (w1, b1), (w2, b2), (w3, b3) = pol._split["actor"]
    assert w1.shape == (2, 8, 32, 4) and w2.shape == (4, 8, 32, 4) and w3.shape == (4, 1, 32, 4)
    assert b1.shape == (64,) and b3.shape == (8,) and float(b3[1:].abs().max()) == 0.0
    # zero rows past in_dim: k-step 1 holds rows 16..31, rows 27..31 are padding -> layer-1 lanes t with 4t+j >= 11 in that k-step
    t = torch.arange(32) % 4
    pad = (4 * t + 2 + 16 >= 28)                                             # second pair (rows 16+4t+2, +3) entirely past row 27
    assert int(w1[1, :, pad, 1].abs().max()) == 0 and int(w1[1, :, pad, 3].abs().max()) == 0
    assert np.isfinite(pol.forward_torch(torch.zeros(3, 27))[0].numpy()).all()


# (in_dim, out_dim): HoverAviary ONE_D_RPM (27, 1), HoverAviary RPM (72, 4), MultiHover RPM D = 2, 3, 8 (144, 8), (216, 12),
# (576, 32), ONE_D_RPM D = 32 (864, 32), and ragged widths that are no multiple of 4 or 16
@pytest.mark.parametrize("in_dim,out_dim", [(27, 1), (72, 4), (144, 8), (216, 12), (576, 32), (864, 32), (5, 1), (49, 8), (131, 12)])
@pytest.mark.parametrize("critic", [True, False])
def test_float64_reference_matches_forward_torch_in_float64(in_dim, out_dim, critic):
    """tests/qs_testlib.PolicyRef (what the GPU tests hold the kernel to) is the network of MlpPolicy.forward_torch: run in
    float64 on the CPU, the two agree to rounding in the last float64 bits."""
    pol = MlpPolicy.random(in_dim, out_dim, seed=in_dim + out_dim, critic=critic, log_std=-0.7, device="cpu")
    ref = PolicyRef(pol)
    g = torch.Generator().manual_seed(3)
    obs = (torch.rand(37, in_dim, generator=g) * 4 - 2).float()
    noise = torch.randn(37, out_dim, generator=g).float()
    p64 = pol.double()
    for nz in (noise, None):
        raw_t, lp_t, v_t = p64.forward_torch(obs.double(), None if nz is None else nz.double())
        assert raw_t.dtype == torch.float64
        mean, raw, lp, v = ref.forward(obs, nz)
        assert np.abs(raw - raw_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(raw).max())
        assert np.abs(lp - lp_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(lp).max())
        if critic:
            assert np.abs(v - v_t.numpy()).max() <= 1e-12 * max(1.0, np.abs(v).max())
        else:
            assert v is None and v_t is None
        if nz is None:
            assert np.array_equal(mean, raw)
    # the fp32 network is the float64 one to fp32 rounding, and the criterion then accepts fp32 itself
    raw32, lp32, v32 = pol.forward_torch(obs, noise)
    r = ref.check(obs, noise, raw32, lp32, v32)
    assert max(r.values()) <= 1.0, r


def test_criterion_floor_is_tanh_error_through_the_following_layers():
    """floor[j] = 6 * 2e-7 sqrt(sum_k W3[k,j]^2 (1 + sum_i W2[i,k]^2)), written out with loops; the worst-case sum of absolute
    values is ~5x larger for 64-unit layers."""
    pol = MlpPolicy.random(20, 3, seed=4, critic=False, device="cpu")
    ref = PolicyRef(pol)
    w2, w3 = ref.actor[1][0], ref.actor[2][0]
    for j in range(3):
        want = 6 * 2e-7 * sum(w3[k, j] ** 2 * (1.0 + sum(w2[i, k] ** 2 for i in range(64))) for k in range(64)) ** 0.5
        assert abs(ref.floor_actor[j] - want) <= 1e-12 * want
        worst = 2e-7 * sum(abs(w3[k, j]) * (1.0 + sum(abs(w2[i, k]) for i in range(64))) for k in range(64))
        assert 3 < worst / ref.floor_actor[j] < 8


def test_fp16_observation_rounding_exceeds_the_criterion():
    """Negative control of the observation operand: a kernel that used only x_hi = fp16(x) would move the actor and the critic
    by far more than the criterion allows.  Observation rows shaped like a MultiHoverAviary RPM one (positions ~1 m, rpy,
    velocities, accelerations, the last 15 actions in [-1, 1])."""
    pol = MlpPolicy.random(144, 8, seed=6, critic=True, device="cpu")
    ref = PolicyRef(pol)
    rng = np.random.default_rng(7)
    x = rng.uniform(-1, 1, (256, 2, 72)).astype(np.float32)
    x[..., :3] *= 2.0
    x[..., 2] += 1.0
    xh = x.astype(np.float16).astype(np.float32)
    mean, raw, lp, v = ref.forward(xh)
    r = ref.check(x, None, raw, lp, v)
    assert r["actions"] > 10 and r["values"] > 10, r


def test_saturation_model():
    """The kernel's observation split saturates at 65504 + 65504 / 2048 in magnitude, not at fp16's 65504: restated in NumPy
    with the same saturating conversions, x_hi + x_lo' / 2048 stops growing at OBS_SATURATION."""
    x = np.array([1.0, 65503.0, 65504.0, 65510.0, 65535.0, 65535.984375, 65536.0, 7e4, 1e6, 3e38], np.float32)
    x = np.concatenate([x, -x])

    def f16sat(v):
        return np.clip(v, -65504.0, 65504.0).astype(np.float16).astype(np.float32)
    hi = f16sat(x)
    with np.errstate(over="ignore"):                         # 3e38 * 2048 is inf in float32, as on the device
        lo = f16sat((x - hi) * np.float32(2048.0))
    seen = hi.astype(np.float64) + lo.astype(np.float64) / 2048.0
    want = PolicyRef.saturate(x)
    assert np.all(np.abs(seen - want) <= 2.0 ** -22 * np.abs(want)), (seen, want)
    assert PolicyRef.OBS_SATURATION == 65535.984375 and seen.max() == PolicyRef.OBS_SATURATION
