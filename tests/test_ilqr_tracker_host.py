"""qs_ctrl_rollout_lqr (the LQR tracker of an iLQR plan in the control rollout) without a GPU: the entry point is exported, the
ctypes mirror of QsLqrRolloutIO has the library's size, every argument refusal comes back as its code and message before anything
is launched, and the float64 restatement tests/ilqr_tracker_ref.py holds on hand-worked cases."""
import ctypes as C

import torch

import ilqr_tracker_ref as TR
from gym_pybullet_drones_b200 import _native as N

ERR_NULL, ERR_ALIGN, ERR_SIZE, ERR_ENUM, ERR_UNSUPPORTED = -1, -2, -3, -4, -5
F64 = torch.float64


def test_entry_point_is_exported_and_the_mirror_matches():
    N.build()
    lib = N.lib()
    assert "qs_ctrl_rollout_lqr" in N.EXPORTS and "qs_sizeof_lqr_rollout_io" in N.EXPORTS
    assert lib.qs_sizeof_lqr_rollout_io() == C.sizeof(N.QsLqrRolloutIO) == 5 * 8 + 4 * 4
    assert lib.qs_abi_version() == N.ABI_VERSION == 4


class _Host:
    """Host memory standing in for device buffers: the refusals are decided before any pointer is dereferenced."""

    def __init__(self):
        self.buf = (C.c_char * 65536)()
        self.base = (C.addressof(self.buf) + 255) & ~255
        self.P, self.st = N.QsParams(), N.QsState()
        self.st.planes, self.st.step_counter, self.st.last_rpm = self.at(0), self.at(8192), self.at(9216)

    def at(self, off):
        return self.base + off

    def io(self, T=4):
        io = N.QsCtrlRolloutIO()
        io.T = T
        return io

    def lio(self, nz=13, T_plan=8, tick0=0, **kw):
        lio = N.QsLqrRolloutIO(K=self.at(16384), z_nom=self.at(32768), rpm_nom=self.at(40960), n_z=nz, T_plan=T_plan, tick0=tick0)
        for k, v in kw.items():
            setattr(lio, k, v)
        return lio

    def call(self, io, lio, E=4, D=2, S=5, eff=0, flags=0):
        lib = N.lib()
        rc = lib.qs_ctrl_rollout_lqr(C.byref(self.P), C.byref(self.st), C.byref(io), C.byref(lio) if lio is not None else None,
                                     E, D, S, eff, flags, None)
        return rc, lib.qs_last_error().decode()


def test_argument_refusals_without_a_gpu():
    h = _Host()
    cases = [
        # (expected code, message fragment, io, lio, kwargs)
        (ERR_NULL, "NULL lio", h.io(), None, {}),
        (ERR_NULL, "NULL K / z_nom / rpm_nom", h.io(), h.lio(K=None), {}),
        (ERR_NULL, "NULL K / z_nom / rpm_nom", h.io(), h.lio(z_nom=None), {}),
        (ERR_NULL, "NULL K / z_nom / rpm_nom", h.io(), h.lio(rpm_nom=None), {}),
        (ERR_SIZE, "n_z must be 13 or 17", h.io(), h.lio(nz=12), {}),
        (ERR_SIZE, "n_z must be 13 or 17", h.io(), h.lio(nz=21), {}),
        (ERR_SIZE, "T_plan must be > 0", h.io(), h.lio(T_plan=0), {}),
        (ERR_SIZE, "T_plan must be > 0", h.io(), h.lio(T_plan=-3), {}),
        (ERR_SIZE, "must lie in the plan", h.io(), h.lio(tick0=-1), {}),
        (ERR_SIZE, "must lie in the plan", h.io(T=4), h.lio(T_plan=8, tick0=5), {}),
        (ERR_SIZE, "must lie in the plan", h.io(T=9), h.lio(T_plan=8), {}),
        (ERR_SIZE, "must be > 0", h.io(T=0), h.lio(), {}),
        (ERR_ALIGN, "32-byte aligned", h.io(), h.lio(rpm_nom=h.at(40960 + 8)), {}),
        (ERR_ALIGN, "32-byte aligned", h.io(), h.lio(lo=h.at(49152 + 16), hi=h.at(53248)), {}),
        (ERR_NULL, "both given or both NULL", h.io(), h.lio(lo=h.at(49152)), {}),
        (ERR_NULL, "both given or both NULL", h.io(), h.lio(hi=h.at(49152)), {}),
        (ERR_SIZE, "per_tick must be 0 or 1", h.io(), h.lio(lo=h.at(49152), hi=h.at(53248), per_tick=2), {}),
        (ERR_UNSUPPORTED, "drones_per_env <= 128", h.io(), h.lio(), dict(E=1, D=129, eff=N.EFFECT_DW)),
        (ERR_UNSUPPORTED, "ACTION_F64 is for QS_CTRL_RAW", h.io(), h.lio(), dict(flags=N.FLAG_ACTION_F64)),
        (ERR_UNSUPPORTED, "GND|DRAG", h.io(), h.lio(), dict(eff=N.EFFECT_GND | N.EFFECT_DRAG)),
    ]
    for code, frag, io, lio, kw in cases:
        rc, msg = h.call(io, lio, **kw)
        assert rc == code and frag in msg, (code, frag, kw, rc, msg)
    io = h.io()
    io.actions = h.at(57344)
    rc, msg = h.call(io, h.lio())
    assert rc == ERR_UNSUPPORTED and "not actions" in msg, msg
    # an n_z = 17 plan needs the previous RPMs; n_z = 13 does not
    h.st.last_rpm = None
    rc, msg = h.call(h.io(), h.lio(nz=17))
    assert rc == ERR_NULL and "needs QsState.last_rpm" in msg, msg
    # the plain entry point does not take the tracker's mode
    rc = N.lib().qs_ctrl_rollout(C.byref(h.P), C.byref(h.st), C.byref(h.io()), N.CTRL_LQR, 4, 2, 5, 0, 0, None)
    assert rc == ERR_ENUM and "bad mode" in N.lib().qs_last_error().decode()


# ---- the restatement on hand-worked cases ------------------------------------------------------------------------------------

def _plan(n=3, nz=13, seed=0):
    g = torch.Generator().manual_seed(seed)
    K = torch.randn((n, 4, nz), generator=g, dtype=F64) * 100.0
    z = torch.randn((n, nz), generator=g, dtype=F64)
    rpm = 14000.0 + 1000.0 * torch.randn((n, 4), generator=g, dtype=F64)
    return K, z, rpm


def test_zero_perturbation_returns_rpm_nom_exactly():
    for nz in (13, 17):
        K, z, rpm = _plan(nz=nz)
        rpm[0, 0] = 0.0                                    # 0.0 + (a sum of signed zeros from 0.0) stays +0.0
        K[:, :, 0] = -K[:, :, 0].abs()                     # negative gains: the products are -0.0
        u = TR.control(z[:, :13], z[:, 13:] if nz == 17 else None, z, K, rpm)
        assert torch.equal(u, rpm)
        assert not torch.signbit(u[0, 0])


def test_clamp_at_each_bound_then_the_motor_clip():
    K = torch.zeros((1, 4, 13), dtype=F64)
    K[0, :, 0] = torch.tensor([1.0, -1.0, 2.0, 0.0], dtype=F64)
    z = torch.zeros((1, 13), dtype=F64)
    x = z.clone()
    x[0, 0] = 1000.0                                       # dz_0 = 1000
    rpm = torch.full((1, 4), 10000.0, dtype=F64)
    lo, hi = torch.full((1, 4), 9500.0, dtype=F64), torch.full((1, 4), 11500.0, dtype=F64)
    assert TR.control(x, None, z, K, rpm).tolist() == [[11000.0, 9000.0, 12000.0, 10000.0]]
    assert TR.control(x, None, z, K, rpm, lo, hi).tolist() == [[11000.0, 9500.0, 11500.0, 10000.0]]
    mr = torch.tensor([10500.0], dtype=F64)
    assert TR.control(x, None, z, K, rpm, lo, hi, max_rpm=mr).tolist() == [[10500.0, 9500.0, 10500.0, 10000.0]]
    x[0, 0] = -20000.0                                     # below 0: the motor clip holds the rotor at 0
    assert TR.control(x, None, z, K, rpm, max_rpm=mr).tolist() == [[0.0, 10500.0, 0.0, 10000.0]]


def test_the_previous_rpms_enter_with_n_z_17():
    K = torch.zeros((1, 4, 17), dtype=F64)
    K[0, 0, 13], K[0, 1, 14], K[0, 2, 15], K[0, 3, 16] = 0.5, -0.25, 1.0, 2.0
    z = torch.zeros((1, 17), dtype=F64)
    z[0, 13:] = torch.tensor([100.0, 200.0, 300.0, 400.0], dtype=F64)
    prev = torch.tensor([[110.0, 180.0, 300.0, 401.0]], dtype=F64)
    rpm = torch.full((1, 4), 1000.0, dtype=F64)
    assert TR.control(z[:, :13], prev, z, K, rpm).tolist() == [[1005.0, 1005.0, 1000.0, 1002.0]]


def test_the_summation_order_is_q_ascending_from_zero():
    # 1 + 2^53 rounds to 2^53 (ties to even), so the order q = 0, 1, 2 gives 0 and the reverse order gives 1
    K = torch.zeros((1, 4, 13), dtype=F64)
    K[0, 0, 0:3] = torch.tensor([1.0, 2.0 ** 53, -(2.0 ** 53)], dtype=F64)
    z = torch.zeros((1, 13), dtype=F64)
    x = z.clone()
    x[0, 0:3] = 1.0
    rpm = torch.full((1, 4), 100.0, dtype=F64)
    assert TR.control(x, None, z, K, rpm)[0, 0].item() == 100.0
    assert TR.control(x, None, z, K, rpm, order=range(12, -1, -1))[0, 0].item() == 101.0
