"""Trajectory logger writing the reference's on-disk format (reference: gym_pybullet_drones/utils/Logger.py:12-127).

Same constructor, `log(drone, timestamp, state, control)`, `save()` and array layout as the reference -- `timestamps`
[D, T], `states` [D, 16, T] in the reference's re-ordered layout (pos3, vel3, rpy3, ang_v3, rpm4; Logger.py:117) and
`controls` [D, 12, T], saved with `np.savez` under the same keys -- so existing analysis scripts keep working.  Added
for the vectorised envs: `log_all(timestamp, states[D, 20], controls[D, 12])` logs every drone of an aviary with one
call, and `attach(env, aviary)`: the env then appends one entry per drone of that aviary after EVERY control tick to a
ring in device memory (qs_log_append: 16 states + 12 controls + time, float64), with no host transfer until `flush()` /
`save()` -- logging a vectorised env no longer costs a D2H copy per tick.  Plotting (`Logger.plot`, Logger.py:205-379)
needs matplotlib, which is optional.
"""
import os
from datetime import datetime

import numpy as np

_REORDER = np.r_[0:3, 10:13, 7:10, 13:20]       # 20-float state vector -> the 16 logged states (Logger.py:117)


class Logger(object):
    def __init__(self, logging_freq_hz: int, output_folder: str = "results", num_drones: int = 1, duration_sec: int = 0, colab: bool = False):
        self.COLAB = colab
        self.OUTPUT_FOLDER = output_folder
        os.makedirs(self.OUTPUT_FOLDER, exist_ok=True)
        self.LOGGING_FREQ_HZ = logging_freq_hz
        self.NUM_DRONES = num_drones
        self.PREALLOCATED_ARRAYS = duration_sec != 0
        n = duration_sec * self.LOGGING_FREQ_HZ
        self.counters = np.zeros(num_drones)
        self.timestamps = np.zeros((num_drones, n))
        self.states = np.zeros((num_drones, 16, n))
        self.controls = np.zeros((num_drones, 12, n))

    def _grow(self, upto):
        have = self.timestamps.shape[1]
        if upto > have:
            extra = max(upto - have, have // 2, 16)
            self.timestamps = np.concatenate((self.timestamps, np.zeros((self.NUM_DRONES, extra))), axis=1)
            self.states = np.concatenate((self.states, np.zeros((self.NUM_DRONES, 16, extra))), axis=2)
            self.controls = np.concatenate((self.controls, np.zeros((self.NUM_DRONES, 12, extra))), axis=2)

    def log(self, drone: int, timestamp, state, control=np.zeros(12)):
        """One entry of one drone (Logger.py:83-119)."""
        state, control = np.asarray(state, dtype=np.float64), np.asarray(control, dtype=np.float64)
        if drone < 0 or drone >= self.NUM_DRONES or timestamp < 0 or len(state) != 20 or len(control) != 12:
            raise ValueError("[ERROR] in Logger.log(), invalid data")
        c = int(self.counters[drone])
        self._grow(c + 1)
        self.timestamps[drone, c] = timestamp
        self.states[drone, :, c] = state[_REORDER]
        self.controls[drone, :, c] = control
        self.counters[drone] = c + 1

    def log_all(self, timestamp, states, controls=None):
        """Every drone of an aviary at once: states [D, 20] (e.g. CtrlAviary observations), controls [D, 12]."""
        states = np.asarray(states, dtype=np.float64).reshape(self.NUM_DRONES, 20)
        c = int(self.counters.max())
        self._grow(c + 1)
        self.timestamps[:, c] = timestamp
        self.states[:, :, c] = states[:, _REORDER]
        if controls is not None:
            self.controls[:, :, c] = np.asarray(controls, dtype=np.float64).reshape(self.NUM_DRONES, 12)
        self.counters[:] = c + 1

    # ---- device-side ring (SURVEY.md 8f rank 4) --------------------------------------------------------------------------
    def attach(self, env, aviary: int = 0, capacity: int = None):
        """Starts logging every control tick of `env`'s aviary `aviary` (its NUM_DRONES drones) on the device.
        `capacity` = ticks the ring holds between two flush() calls (default: duration_sec * logging_freq_hz, else 4096).
        The ring records the env's storage slots, so an env whose storage `reorder_by_morton()` has permuted is refused
        (ValueError), and so is a reorder while a Logger is attached; log such a formation with `log_all` and its observations."""
        import ctypes as C
        import torch
        from .. import _native as N
        if env.NUM_DRONES != self.NUM_DRONES:
            raise ValueError("Logger(num_drones=%d) attached to an env with %d drones per aviary" % (self.NUM_DRONES, env.NUM_DRONES))
        if getattr(env, "_order", None) is not None:
            raise ValueError("Logger.attach() on an env reordered by reorder_by_morton(): the device ring records storage slots, "
                             "not drone ids; log its observations with log_all() instead")
        if not 0 <= aviary < env.num_envs:
            raise ValueError("aviary index out of range")
        cap = int(capacity or (self.timestamps.shape[1] if self.PREALLOCATED_ARRAYS else 4096))
        self._ring = torch.zeros((cap, self.NUM_DRONES, 32), dtype=torch.float64, device=env.device)
        self._head = torch.zeros((1,), dtype=torch.int64, device=env.device)
        self._ctrl_dev = torch.zeros((self.NUM_DRONES, 12), dtype=torch.float32, device=env.device)
        rg = N.QsLogRing()
        rg.ring, rg.head, rg.capacity = self._ring.data_ptr(), self._head.data_ptr(), cap
        rg.first_drone, rg.n_drones = aviary * env.NUM_DRONES, self.NUM_DRONES
        rg.kin_rows = 0 if env._state20_obs() else 1          # a KIN row can be 20 floats wide as well
        self._rg, self._env, self._flushed = rg, env, 0
        env._log = (rg, self._ctrl_dev)
        return self

    def set_controls(self, controls):
        """Control targets [D, 12] logged with the following ticks (Logger.py:59-72); ndarray or CUDA tensor."""
        import torch
        c = controls if isinstance(controls, torch.Tensor) else torch.as_tensor(np.asarray(controls, dtype=np.float32))
        self._ctrl_dev.copy_(c.to(dtype=torch.float32).reshape(self.NUM_DRONES, 12), non_blocking=True)

    def detach(self):
        self.flush()
        self._env._log = None
        self._env = None

    def flush(self):
        """Copies the entries appended since the last flush from the device ring into the host arrays (one D2H)."""
        if getattr(self, "_env", None) is None:
            return 0
        head = int(self._head.item())
        cap = self._rg.capacity
        n_new = head - self._flushed
        if n_new <= 0:
            return 0
        if n_new > cap:
            raise RuntimeError("Logger ring overflow: %d ticks since the last flush(), capacity %d" % (n_new, cap))
        idx = np.arange(self._flushed, head) % cap
        rows = self._ring.cpu().numpy()[idx]                  # [n_new, D, 32]
        c = int(self.counters.max())
        self._grow(c + n_new)
        self.timestamps[:, c:c + n_new] = rows[:, :, 28].T
        self.states[:, :, c:c + n_new] = rows[:, :, 0:16].transpose(1, 2, 0)
        self.controls[:, :, c:c + n_new] = rows[:, :, 16:28].transpose(1, 2, 0)
        self.counters[:] = c + n_new
        self._flushed = head
        return n_new

    def _trimmed(self):
        n = int(self.counters.max()) if not self.PREALLOCATED_ARRAYS else self.timestamps.shape[1]
        return self.timestamps[:, :n], self.states[:, :, :n], self.controls[:, :, :n]

    def save(self):
        """np.savez(timestamps=, states=, controls=) like the reference (Logger.py:123-127); returns the path."""
        self.flush()
        ts, st, ct = self._trimmed()
        path = os.path.join(self.OUTPUT_FOLDER, "save-flight-" + datetime.now().strftime("%m.%d.%Y_%H.%M.%S") + ".npy")
        with open(path, 'wb') as out_file:
            np.savez(out_file, timestamps=ts, states=st, controls=ct)
        return path

    def save_as_csv(self, comment: str = ""):
        """One two-column CSV (time, value) per drone and signal, named like the reference's (Logger.py:131-201)."""
        ts, st, _ = self._trimmed()
        folder = os.path.join(self.OUTPUT_FOLDER, "save-flight-" + comment + "-" + datetime.now().strftime("%m.%d.%Y_%H.%M.%S"))
        os.makedirs(folder, exist_ok=True)
        names = ["x", "y", "z", "vx", "vy", "vz", "r", "p", "ya", "wx", "wy", "wz", "rpm0", "rpm1", "rpm2", "rpm3"]
        for i in range(self.NUM_DRONES):
            for k, nm in enumerate(names):
                np.savetxt(os.path.join(folder, "%s%d.csv" % (nm, i)), np.stack([ts[i], st[i, k]], axis=1), delimiter=",")
        return folder

    def plot(self, pwm=False):
        try:
            import matplotlib.pyplot as plt
        except Exception as e:  # pragma: no cover
            raise ImportError("Logger.plot needs matplotlib, which is not installed") from e
        ts, st, _ = self._trimmed()
        fig, axs = plt.subplots(8, 2)
        labels = ["x (m)", "y (m)", "z (m)", "vx (m/s)", "vy (m/s)", "vz (m/s)", "r (rad)", "p (rad)", "y (rad)", "wx", "wy", "wz", "RPM0", "RPM1", "RPM2", "RPM3"]
        for k in range(16):
            ax = axs[k % 8, k // 8]
            for j in range(self.NUM_DRONES):
                ax.plot(ts[j], st[j, k], label="drone_" + str(j))
            ax.set_ylabel(labels[k]); ax.grid(True)
        if not self.COLAB:
            plt.show()
        return fig
