"""Float64 torch restatement of the LQR tracker of qs_ctrl_rollout_lqr (include/quadsim.h, DESIGN.md 4.1e) in the kernel's order of
operations: dz = (x - z_nom[0:13], rpm_prev - z_nom[13:17]); s_j = sum_q K_jq dz_q summed from 0.0 in the order q = 0, 1, ...;
u_j = rpm_nom_j + s_j; u = clampd(u, lo, hi) with bounds; then the env's clampd(u, 0, MAX_RPM).  Every step is one rounded float64
operation, as in the kernel (built with -fmad=false), so the result is the kernel's bits."""
import torch

KEYS = ("pos", "quat", "vel", "rpy_rates")


def clampd(v, lo, hi):
    """qs::clampd: v < lo ? lo : (v > hi ? hi : v)"""
    lo, hi = torch.as_tensor(lo, dtype=v.dtype, device=v.device), torch.as_tensor(hi, dtype=v.dtype, device=v.device)
    return torch.where(v < lo, lo, torch.where(v > hi, hi, v))


def drone_vec(planes, n):
    """[13 N] planes -> [N, 13] in drone_vec's order (px py pz qx qy qz qw vx vy vz wx wy wz)"""
    from gym_pybullet_drones_b200.diff import unpack_states
    u = unpack_states(planes, n)
    return torch.cat([u[k] for k in KEYS], dim=-1)


def control(x, rpm_prev, z_nom, K, rpm_nom, lo=None, hi=None, max_rpm=None, order=None):
    """The applied RPMs [N, 4] of one tick: x [N, 13] the state, rpm_prev [N, 4] the RPMs applied at the tick before, z_nom
    [N, n_z], K [N, 4, n_z], rpm_nom [N, 4], lo / hi [N, 4] or None, max_rpm [N] (None: no clip).  `order` permutes the
    summation (negative controls)."""
    nz = K.shape[-1]
    dz = x - z_nom[:, :13]
    if nz == 17:
        dz = torch.cat([dz, rpm_prev - z_nom[:, 13:]], dim=1)
    order = range(nz) if order is None else order
    u = torch.empty_like(rpm_nom)
    for j in range(4):
        s = torch.zeros_like(rpm_nom[:, j])
        for q in order:
            s = s + K[:, j, q] * dz[:, q]
        u[:, j] = rpm_nom[:, j] + s
    if lo is not None:
        u = clampd(u, lo, hi)
    if max_rpm is not None:
        u = clampd(u, torch.zeros_like(u), max_rpm.reshape(-1, 1).expand_as(u))
    return u
