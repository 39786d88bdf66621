"""qs_ctrl_rollout (the control envs' T-tick rollout) at the C ABI, without a GPU: the entry point is exported, the ctypes mirror
of QsCtrlRolloutIO has the library's size, every argument refusal comes back as its code and message before anything is
launched, and the NumPy restatement of the waypoint rule matches a hand-worked schedule."""
import ctypes as C

import numpy as np

from gym_pybullet_drones_b200 import _native as N
from gym_pybullet_drones_b200.envs.CtrlAviary import CtrlAviary

ERR_NULL, ERR_ALIGN, ERR_SIZE, ERR_ENUM, ERR_UNSUPPORTED = -1, -2, -3, -4, -5


def test_entry_point_is_exported_and_the_mirror_matches():
    N.build()
    lib = N.lib()
    assert "qs_ctrl_rollout" in N.EXPORTS and "qs_sizeof_ctrl_rollout_io" in N.EXPORTS
    assert getattr(lib, "qs_ctrl_rollout") is not None
    assert lib.qs_sizeof_ctrl_rollout_io() == C.sizeof(N.QsCtrlRolloutIO)
    assert lib.qs_abi_version() == N.ABI_VERSION == 4


class _Host:
    """Host memory standing in for device buffers: the refusals are decided before any pointer is dereferenced."""

    def __init__(self):
        self.buf = (C.c_char * 65536)()
        self.base = (C.addressof(self.buf) + 255) & ~255
        self.P, self.CP, self.st = N.QsParams(), N.QsParams(), N.QsState()
        self.st.planes, self.st.step_counter, self.st.last_rpm, self.st.pid = self.at(0), self.at(8192), self.at(9216), self.at(10240)
        self.ring = N.QsLogRing()

    def at(self, off):
        return self.base + off

    def raw(self, T=4):
        io = N.QsCtrlRolloutIO()
        io.T, io.actions = T, self.at(16384)
        return io

    def track(self, T=4):
        io = N.QsCtrlRolloutIO()
        io.T = T
        io.ctrl_params, io.pid_state, io.control_timestep = C.addressof(self.CP), self.at(20480), 1 / 48
        io.waypoints, io.W, io.M, io.start = self.at(24576), 8, 1, self.at(28672)
        return io

    def call(self, io, mode=N.CTRL_RAW, E=4, D=2, S=5, eff=0, flags=0, p=True, st=True):
        lib = N.lib()
        rc = lib.qs_ctrl_rollout(C.byref(self.P) if p else None, C.byref(self.st) if st else None, C.byref(io) if io is not None else None,
                                 mode, E, D, S, eff, flags, None)
        return rc, lib.qs_last_error().decode()


def test_argument_refusals_without_a_gpu():
    h = _Host()
    cases = [
        # (expected code, message fragment, io, kwargs)
        (ERR_NULL, "NULL params/io", h.raw(), dict(p=False)),
        (ERR_NULL, "NULL params/io", None, {}),
        (ERR_NULL, "planes", h.raw(), dict(st=False)),
        (ERR_SIZE, "must be > 0", h.raw(T=0), {}),
        (ERR_SIZE, "must be > 0", h.raw(), dict(E=0)),
        (ERR_SIZE, "must be > 0", h.raw(), dict(S=0)),
        (ERR_SIZE, "2^31-1", h.raw(), dict(E=1 << 20, D=1 << 12)),
        (ERR_ENUM, "bad mode", h.raw(), dict(mode=3)),
        (ERR_ENUM, "bad effects", h.raw(), dict(eff=8)),
        (ERR_UNSUPPORTED, "GND|DRAG", h.raw(), dict(eff=N.EFFECT_GND | N.EFFECT_DRAG)),
        (ERR_UNSUPPORTED, "drones_per_env <= 128", h.raw(), dict(E=1, D=129, eff=N.EFFECT_DW)),
        (ERR_UNSUPPORTED, "drones_per_env <= 128", h.raw(), dict(E=1, D=129, eff=7)),
        (ERR_UNSUPPORTED, "only QS_FLAG_RPY_F32", h.raw(), dict(flags=N.FLAG_AUTORESET_SAME_STEP)),
        (ERR_UNSUPPORTED, "only QS_FLAG_RPY_F32", h.raw(), dict(flags=N.FLAG_OBS_STATE20)),
        (ERR_UNSUPPORTED, "ACTION_F64 is for QS_CTRL_RAW", h.raw(), dict(mode=N.CTRL_VEL, flags=N.FLAG_ACTION_F64)),
        (ERR_UNSUPPORTED, "not actions", h.raw(), dict(mode=N.CTRL_TRACK)),
    ]
    for code, frag, io, kw in cases:
        rc, msg = h.call(io, **kw)
        assert rc == code and frag in msg, (code, frag, kw, rc, msg)
    # misaligned state planes
    st_planes = h.st.planes
    h.st.planes = h.at(8)
    rc, msg = h.call(h.raw())
    assert rc == ERR_ALIGN and "planes" in msg
    h.st.planes = st_planes
    # actions: NULL, float32 16-byte, float64 32-byte alignment
    io = h.raw()
    io.actions = None
    assert h.call(io) == (ERR_NULL, "qs_ctrl_rollout: actions is NULL")
    io.actions = h.at(16384 + 8)
    assert h.call(io)[0] == ERR_ALIGN
    io.actions = h.at(16384 + 16)
    rc, msg = h.call(io, flags=N.FLAG_ACTION_F64)
    assert rc == ERR_ALIGN and "32-byte" in msg
    # outputs: rpm 32-byte, obs / obs_last 16-byte
    io = h.raw()
    io.rpm = h.at(32768 + 16)
    assert h.call(io)[0] == ERR_ALIGN and "rpm" in h.call(io)[1]
    io = h.raw()
    io.obs = h.at(32768 + 4)
    assert h.call(io)[0] == ERR_ALIGN
    io = h.raw()
    io.obs_last = h.at(32768 + 8)
    assert h.call(io)[0] == ERR_ALIGN
    # VEL needs the embedded controller's state
    pid = h.st.pid
    h.st.pid = None
    rc, msg = h.call(h.raw(), mode=N.CTRL_VEL)
    assert rc == ERR_NULL and "QsState.pid" in msg
    h.st.pid = pid
    # DRAG needs last_rpm
    lr = h.st.last_rpm
    h.st.last_rpm = None
    rc, msg = h.call(h.raw(), eff=N.EFFECT_DRAG)
    assert rc == ERR_NULL and "last_rpm" in msg
    h.st.last_rpm = lr


def test_track_refusals_without_a_gpu():
    h = _Host()
    io = h.track()
    io.ctrl_params = None
    rc, msg = h.call(io, mode=N.CTRL_TRACK)
    assert rc == ERR_NULL and "needs a controller" in msg
    io = h.track()
    io.pid_state = None
    assert h.call(io, mode=N.CTRL_TRACK)[0] == ERR_NULL
    io = h.track()
    io.waypoints = None
    rc, msg = h.call(io, mode=N.CTRL_TRACK)
    assert rc == ERR_NULL and "waypoints" in msg
    io = h.track()
    io.start = None
    assert h.call(io, mode=N.CTRL_TRACK)[0] == ERR_NULL
    for W in (0, -3):
        io = h.track()
        io.W = W
        rc, msg = h.call(io, mode=N.CTRL_TRACK)
        assert rc == ERR_SIZE and "W (waypoint rows)" in msg
    io = h.track()
    io.M = 3                                                    # neither 1 nor N = 8
    rc, msg = h.call(io, mode=N.CTRL_TRACK)
    assert rc == ERR_SIZE and "M (waypoint columns)" in msg
    io = h.track()
    io.control_timestep = 0.0
    assert h.call(io, mode=N.CTRL_TRACK)[0] == ERR_SIZE
    # the log ring
    io = h.track()
    io.log = C.addressof(h.ring)
    rc, msg = h.call(io, mode=N.CTRL_TRACK)
    assert rc == ERR_NULL and "log ring" in msg
    h.ring.ring, h.ring.head, h.ring.capacity, h.ring.first_drone, h.ring.n_drones = h.at(40960), h.at(49152), 16, 6, 4
    rc, msg = h.call(io, mode=N.CTRL_TRACK)                     # drones 6..9 of 8
    assert rc == ERR_SIZE and "ring geometry" in msg


def test_waypoint_rule_restatement_matches_a_hand_worked_case():
    # W = 4 shared waypoints, three drones with phases 0, 3, -1 (Python's mod: -1 -> row 3), offsets lift each drone's z
    wp = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [1.0, 1.0, 0.0], [0.0, 1.0, 0.0]])
    start = np.array([0, 3, -1])
    offset = np.array([[0.0, 0.0, 0.1], [0.0, 0.0, 0.2], [10.0, 0.0, 0.3]])
    tp = CtrlAviary.schedule_targets(wp, start, offset, 3)
    want = np.array([
        [[0.0, 0.0, 0.1], [0.0, 1.0, 0.2], [10.0, 1.0, 0.3]],         # k = 0: rows 0, 3, 3
        [[1.0, 0.0, 0.1], [0.0, 0.0, 0.2], [10.0, 0.0, 0.3]],         # k = 1: rows 1, 0, 0
        [[1.0, 1.0, 0.1], [1.0, 0.0, 0.2], [11.0, 0.0, 0.3]],         # k = 2: rows 2, 1, 1
    ])
    assert tp.shape == (3, 3, 3) and np.array_equal(tp, want)
    # per-drone paths (M = n): drone i reads column i; W = T is a full schedule
    per = np.arange(2 * 3 * 3, dtype=np.float64).reshape(2, 3, 3)
    tp = CtrlAviary.schedule_targets(per, [0, 1, 2], None, 2)
    assert np.array_equal(tp[0], np.stack([per[0, 0], per[1, 1], per[0, 2]]))
    assert np.array_equal(tp[1], np.stack([per[1, 0], per[0, 1], per[1, 2]]))
