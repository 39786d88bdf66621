"""The C-ABI library loads on a machine without a GPU and exports every symbol include/quadsim.h declares; the ctypes
mirrors have the library's struct sizes; argument validation works without launching anything."""
import ctypes as C
import os
import re

from gym_pybullet_drones_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "quadsim.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(qs_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    N.build()                                   # no-op when the in-tree .so is newer than its sources
    lib = N.lib()
    syms = declared_symbols()
    assert len(syms) >= 14 and set(N.EXPORTS) == set(syms)
    for s in syms:
        assert getattr(lib, s) is not None, s
    assert lib.qs_abi_version() == N.ABI_VERSION


def test_struct_mirrors_match_the_library():
    lib = N.lib()
    assert lib.qs_sizeof_params() == C.sizeof(N.QsParams) and lib.qs_sizeof_state() == C.sizeof(N.QsState)
    assert lib.qs_sizeof_step_io() == C.sizeof(N.QsStepIO) and lib.qs_sizeof_rollout_io() == C.sizeof(N.QsRolloutIO)
    assert lib.qs_sizeof_host_io() == C.sizeof(N.QsHostIO)


def test_argument_errors_without_a_gpu():
    """Every entry point validates its arguments before touching CUDA: negative codes + a message, no launch."""
    lib = N.lib()
    P, st, io = N.QsParams(), N.QsState(), N.QsStepIO()
    assert lib.qs_step(None, C.byref(st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, None) == -1
    assert lib.qs_step(C.byref(P), C.byref(st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, None) == -1          # NULL planes
    assert b"planes" in lib.qs_last_error()
    buf = (C.c_float * 64)()
    st.planes = C.addressof(buf) + 4
    st.step_counter = C.addressof(buf)
    assert lib.qs_step(C.byref(P), C.byref(st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, None) == -2          # misaligned planes
    assert lib.qs_rollout_max_ticks(N.ACT_RPM, 15, 2) == 255 and lib.qs_rollout_max_ticks(N.ACT_RPM, 120, 2) == 0
    assert lib.qs_rollout_max_ticks(N.ACT_ONE_D_RPM, 15, 1) > 1000 and lib.qs_rollout_max_ticks(99, 15, 1) == 0
    assert lib.qs_pid_control(C.byref(P), None, 0.01, None, 3, None, 4, None, 3, None, None, None, None, 8, None, None, None, None) == -1
    assert lib.qs_downwash(C.byref(P), C.byref(st), 0, 4, None, None) == -1
    assert lib.qs_reset(C.byref(P), C.byref(st), None, 1, 1, 0, None, 12, 0, None) == -2
    try:
        N.check(-3, "x")
        raise AssertionError("check() must raise")
    except ValueError:
        pass


def test_header_is_plain_c99():
    """include/quadsim.h is the drop-in boundary: it must compile as C (what cgo / JNI / ctypes-style bindings see), not
    only as C++."""
    import subprocess
    h = os.path.join(ROOT, "include", "quadsim.h")
    for cmd in (["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", h],
                ["g++", "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++", h]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_formation_entry_points_validate_arguments():
    lib = N.lib()
    P = N.QsParams()
    buf = (C.c_float * 256)()
    a = C.addressof(buf)
    a16 = (a + 15) & ~15
    assert lib.qs_dw_gathered_floats(0) == 0 and lib.qs_dw_gathered_floats(33) == 4 * 33 + 8 * 2
    assert lib.qs_dw_boxes(None, 8, None) == -1 and lib.qs_dw_boxes(a16 + 4, 8, None) == -2 and lib.qs_dw_boxes(a16, 0, None) == -3
    assert lib.qs_downwash_rows(C.byref(P), a16, 8, None, 8, None, 0, 0, None, a16, None) == -1
    assert lib.qs_downwash_rows(C.byref(P), a16, 8, a16, 8, a16, 1, 17, None, a16, None) == -3          # world > QS_MAX_PEERS
    g = (C.c_void_p * 2)(a16, a16)
    f = (C.c_void_p * 2)(a16, a16)
    assert lib.qs_dw_publish(a16, 64, 16, g, 128, f, 2, 0, 1, a16, None) == -2                          # offset not a multiple of 32
    assert b"multiple of 32" in lib.qs_last_error()
    assert lib.qs_dw_publish(a16, 40, 0, g, 128, f, 2, 0, 1, a16, None) == -2                           # a chunk would straddle ranks
    assert lib.qs_dw_publish(a16, 64, 96, g, 128, f, 2, 0, 1, a16, None) == -3                          # slice beyond n_total
    assert lib.qs_dw_publish(a16, 64, 0, g, 128, f, 2, 2, 1, a16, None) == -3                           # rank outside world
    st = N.QsState()
    assert lib.qs_adjacency(C.byref(st), 1, 4, 1.0, None, None) == -1
    assert lib.qs_downwash_boxed(C.byref(P), C.byref(st), 1, 4, None, None, None) == -1
    off = C.c_ulonglong(0)
    assert lib.qs_ipc_export(None, buf, C.byref(off)) == -1 and lib.qs_ipc_import(None, 0, None) == -1


def test_product_package_does_not_import_the_oracle():
    """The oracle is test infrastructure: nothing under the product package may reference it."""
    pkg = os.path.join(ROOT, "gym_pybullet_drones_b200")
    for base, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(base, f)).read()
                assert "oracle" not in src.replace("oracle/", "").replace("the oracle", "") or "import oracle" not in src and "from oracle" not in src, f
                assert "import oracle" not in src and "from oracle" not in src, f


def test_round2_entry_points_validate_arguments_without_a_gpu():
    """qs_pid_control_state / qs_log_append / qs_wait_flags / qs_reset_heads / the policy of qs_rollout / obs_gather of qs_step:
    argument errors come back as negative codes with a message, nothing is launched."""
    lib = N.lib()
    P, st = N.QsParams(), N.QsState()
    assert lib.qs_pid_control_state(C.byref(P), None, 0.02, C.byref(st), 4, None, None, None, None, None, None, None, None) == -1
    assert lib.qs_wait_flags(None, 1, 2, None, None) == -1 and b"flags" in lib.qs_last_error()
    buf = (C.c_char * 4096)()
    base = (C.addressof(buf) + 63) & ~63
    assert lib.qs_wait_flags(base, 1, 99, None, None) == -3
    assert lib.qs_reset_heads(C.byref(st), 4, 0, None, None) == -1
    ring = N.QsLogRing()
    assert lib.qs_log_append(C.byref(P), C.byref(st), base, 20, None, C.byref(ring), 1, 4, None) == -1
    assert lib.qs_sizeof_log_ring() == C.sizeof(N.QsLogRing)
    assert lib.qs_host_is_pinned(None) == 0
    # obs_gather needs a configuration of the fast kernels and 16-byte alignment
    io = N.QsStepIO()
    st.planes, st.step_counter = base, base + 2048
    st.target_pos = base + 1024
    io.action, io.obs_prev, io.obs = base + 256, base + 512, base + 768
    io.reward, io.terminated, io.truncated = base + 1280, base + 1536, base + 1600
    io.act_buffer_size = 15
    io.obs_gather = base + 3000 + 4                                    # misaligned
    assert lib.qs_step(C.byref(P), C.byref(st), C.byref(io), 0, 1, 4, 1, 8, 0, 0, None) == -2
    io.obs_gather = base + 3008
    assert lib.qs_step(C.byref(P), C.byref(st), C.byref(io), 1, 1, 4, 1, 8, 0, 0, None) in (-1, -5)   # PID action: not a fast-kernel configuration
    # the on-device policy: RPM / ONE_D_RPM only, complete actor, matching widths
    rio, pol = N.QsRolloutIO(), N.QsPolicy()
    rio.obs_init, rio.obs, rio.reward, rio.terminated, rio.truncated = base + 512, base + 768, base + 1280, base + 1536, base + 1600
    rio.T, rio.act_buffer_size = 4, 15
    rio.policy = C.addressof(pol)
    assert lib.qs_rollout(C.byref(P), C.byref(st), C.byref(rio), 0, 1, 4, 2, 8, 0, 0, None) == -1 and b"policy" in lib.qs_last_error()
    assert lib.qs_last_error().startswith(b"qs_rollout: ")


def test_fused_publish_entry_point_validates_arguments_without_a_gpu():
    """qs_dyn_substeps_pub (formation exchange fused into the dynamics launch): argument errors come back as negative codes with
    a message, nothing is launched; pub == NULL is plain qs_dyn_substeps."""
    lib = N.lib()
    P, st = N.QsParams(), N.QsState()
    buf = (C.c_char * 8192)()
    base = (C.addressof(buf) + 63) & ~63
    st.planes, st.step_counter = base, base + 4096
    rpm = base + 1024
    pub = N.QsDwPublish()
    call = lambda n_envs, D, pb: lib.qs_dyn_substeps_pub(C.byref(P), C.byref(st), rpm, None, None, n_envs, D, 1, 0, 0, pb, None)
    assert call(1, 64, C.byref(pub)) == -1 and b"publish pointer" in lib.qs_last_error()             # NULL gathered / flags / counter
    g = (C.c_void_p * 2)(base + 2048, base + 2048)
    f = (C.c_void_p * 2)(base + 3072, base + 3072)
    pub.gathered, pub.flags, pub.counter = g, f, base + 3584
    pub.n_total, pub.world, pub.rank, pub.offset, pub.seq = 128, 17, 0, 0, 1
    assert call(1, 64, C.byref(pub)) == -3                                                           # world > QS_MAX_PEERS
    pub.world, pub.rank = 2, 2
    assert call(1, 64, C.byref(pub)) == -3                                                           # rank outside world
    pub.rank = 0
    assert call(2, 32, C.byref(pub)) == -5 and b"one aviary" in lib.qs_last_error()                  # one formation = one aviary
    pub.offset = 96
    assert call(1, 64, C.byref(pub)) == -3                                                           # slice beyond n_total
    pub.offset = 16
    assert call(1, 64, C.byref(pub)) == -2 and b"multiple of 32" in lib.qs_last_error()              # a chunk would straddle ranks
    pub.offset = 0
    assert call(1, 40, C.byref(pub)) == -2                                                           # ragged slice that is not the last one
    g[1] = None
    assert call(1, 64, C.byref(pub)) == -1 and b"peer pointer" in lib.qs_last_error()
    g[1] = base + 2048 + 4
    assert call(1, 64, C.byref(pub)) == -2 and b"16-byte" in lib.qs_last_error()
