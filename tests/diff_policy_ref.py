"""Float64 torch restatement of the policy loop of BaseAviary.differentiable_rollout(policy=) (DESIGN.md 4.5): the KIN observation
built from the state, the MlpPolicy actor, the action clip, the history buffer, the RPM / ONE_D_RPM decode and diff_ref's tick.
Its autograd is the reference gradient of qs_dyn_policy_traj_vjp (test infrastructure, CPU or CUDA tensors).

The decisions: the action clip is torch.clamp; ReLU is torch.relu; the Euler angles are differentiated on the branch of the gimbal
guard the forward takes (diff_pid_ref.quat_to_euler); ang_v = R_last w with R_last = I + 2 (2 - |q|^2) M(q) of the attitude at the
start of the tick's last substep (of the normalised initial attitude for the first observation).  `flip` names decisions to turn
the other way -- negative controls only: "history" cuts the gradient through the buffered actions, "clip" passes it straight
through the action clip, "relu" treats every ReLU unit as alive."""
import math

import torch

import diff_pid_ref as PR
import diff_ref as R


def matrix_unit(q):
    """quat_to_matrix_unit: [B, 3, 3] with s = 2 (2 - |q|^2)."""
    x, y, z, w = q.unbind(1)
    s = 2.0 * (2.0 - (x * x + y * y + z * z + w * w))
    return torch.stack([1 - s * (y * y + z * z), s * (x * y - w * z), s * (x * z + w * y),
                        s * (x * y + w * z), 1 - s * (x * x + z * z), s * (y * z - w * x),
                        s * (x * z - w * y), s * (y * z + w * x), 1 - s * (x * x + y * y)], dim=1).reshape(-1, 3, 3)


def tick(K, rows, x, rpm, up, S, effects):
    """diff_ref.tick that also returns the attitude at the start of the last substep."""
    mx = rows[:, 13:14].expand_as(rpm)
    u = torch.clamp(rpm, min=torch.zeros_like(rpm), max=mx)
    q = x[:, 3:7]
    x = torch.cat([x[:, 0:3], q / torch.sqrt((q * q).sum(1, keepdim=True)), x[:, 7:13]], dim=1)
    k = 2 * math.pi
    ds_prev, ds_cur = (k * up / 60).sum(1), (k * u / 60).sum(1)
    for s in range(S):
        ql = x[:, 3:7]
        x = R.substep(K, rows, x, u, ds_prev if s == 0 else ds_cur, effects)
    return x, u, ql


def actor(theta, activation, obs, flip=()):
    h = obs
    for k in range(0, len(theta) - 3, 2):
        z = h @ theta[k] + theta[k + 1]
        if activation == "tanh":
            h = torch.tanh(z)
        else:
            h = torch.relu(z)
            if "relu" in flip:
                h = z + (h - z).detach()
    return h @ theta[-3] + theta[-2]


def one_tick(K, rows, theta, activation, x, ql, hist, up, noise_k, E, D, S, effects, flip=()):
    """One tick from x [n, 13], the attitude ql [n, 4] whose matrix_unit is R_last, the buffer hist [n, B, A] and the previous
    clipped rpm up.  Returns (x', u, ql', raw [n, A], obs [E, D * od], hist')."""
    n, B, A = hist.shape
    ang = (matrix_unit(ql) @ x[:, 10:13, None])[:, :, 0]
    h = hist.detach() if "history" in flip else hist
    obs = torch.cat([x[:, 0:3], PR.quat_to_euler(x[:, 3:7]), x[:, 7:10], ang, h.reshape(n, B * A)], dim=1).reshape(E, -1)
    raw = actor(theta, activation, obs, flip)
    if noise_k is not None:
        raw = raw + torch.exp(theta[-1]) * noise_k
    raw = raw.reshape(n, A)
    a = torch.clamp(raw, -1.0, 1.0)
    if "clip" in flip:
        a = raw + (a - raw).detach()
    hist = torch.cat([hist[:, 1:], a[:, None, :]], dim=1)
    rpm = (rows[:, 12:13] * (1.0 + 0.05 * a)).expand(n, 4)
    x, u, ql = tick(K, rows, x, rpm, up, S, effects)
    return x, u, ql, raw, obs, hist


def policy_loop(K, rows, theta, activation, x0, abuf, last_rpm, noise, T, E, D, S, effects, flip=()):
    """T ticks for n = E * D drones from x0 [n, 13] and the action buffer abuf [n, B, A] (oldest first), rows [n, 16] per drone,
    theta = [W1, b1, ..., Wout, bout, log_std], noise [T, E, D * A] or None.  Returns (states [T, n, 13], raw actions [T, n, A],
    obs [T, E, D * od])."""
    x, up, hist = x0, last_rpm, abuf
    q0 = x0[:, 3:7]
    ql = q0 / torch.sqrt((q0 * q0).sum(1, keepdim=True))
    xs, raws, obss = [], [], []
    for k in range(T):
        x, up, ql, raw, obs, hist = one_tick(K, rows, theta, activation, x, ql, hist, up, None if noise is None else noise[k], E, D, S,
                                             effects, flip)
        xs.append(x); raws.append(raw); obss.append(obs)
    return torch.stack(xs), torch.stack(raws), torch.stack(obss)
