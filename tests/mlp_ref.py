"""The float64 reference and accuracy criterion of tests/qs_testlib.PolicyRef, generalised to every network the on-device policy
accepts (MlpPolicy: 1 to 4 hidden layers, any widths up to the cap, Tanh or ReLU, separate actor and critic shapes)."""
import numpy as np

from qs_testlib import PolicyRef


class MlpRef(PolicyRef):
    """PolicyRef for any depth and activation.  The criterion is PolicyRef's:
        |kernel - float64| <= FP32_MULTIPLE * e32[j] + floor[j]
    with e32 the error of the same network in NumPy float32 at these inputs.  The floor carries tanh_fast's absolute error e
    through the network as a root sum of squares, in units of e^2 per hidden unit:
        v_0[k] = a,   v_l[k] = a + sum_i W_l[i, k]^2 v_(l-1)[i],   floor[j] = TANH_SIGMAS * e * sqrt(sum_k W_L[k, j]^2 v_(L-1)[k])
    where a = 1 for Tanh (each unit adds its own error; tanh' <= 1 passes the incoming one on) and a = 0 for ReLU (exact, slope
    <= 1).  For [64, 64] Tanh this is PolicyRef._floor term by term.  `activation` overrides the policy's (negative controls).

    ReLU networks get one more term, because e32 alone is no yardstick when the batch has no spread: in a deterministic rollout
    every aviary of a fresh env sees the same observation, fp32 may round that one row almost exactly, and a tolerance of 16 e32
    then rejects the kernel's ordinary operand-split error (measured: up to 8.5x on H100).  Each product of the kernel carries
    at most SPLIT_REL = 2^-21 relative error, so a unit's pre-activation has a standard deviation of at most
    SPLIT_REL sqrt(sum_i (h_i W[i, k])^2), which passes on through ReLU (slope <= 1) and the following layers as a root sum of
    squares, row by row, scaled by TANH_SIGMAS.  With Tanh the activation floor above is the larger term (|h| <= 1), so Tanh
    keeps PolicyRef's criterion unchanged."""
    SPLIT_REL = 2.0 ** -21

    def __init__(self, pol, activation=None):
        self.activation = activation or pol.activation
        super().__init__(pol)

    def tolerance(self, net, floor, x):
        y64, tol = super().tolerance(net, floor, x)
        if self.activation != "relu":
            return y64, tol
        h = np.asarray(x).astype(np.float64)
        var = np.zeros_like(h)
        for k, (w, b) in enumerate(net):
            w2 = w ** 2
            var = self.SPLIT_REL ** 2 * ((h ** 2) @ w2) + var @ w2
            h = h @ w + b
            if k < len(net) - 1:
                h = np.maximum(h, 0.0)
        return y64, tol + self.TANH_SIGMAS * np.sqrt(var)

    def _floor(self, net):
        a = 1.0 if self.activation == "tanh" else 0.0
        v = np.full(net[0][0].shape[1], a)
        for w, _ in net[1:-1]:
            v = (w ** 2 * v[:, None]).sum(axis=0) + a
        return self.TANH_SIGMAS * self.TANH_FAST_ABS_ERR * np.sqrt((net[-1][0] ** 2 * v[:, None]).sum(axis=0))

    def mlp(self, net, x, dtype=np.float64):
        act = np.tanh if self.activation == "tanh" else (lambda h: np.maximum(h, dtype(0)))
        h = np.asarray(x).astype(dtype)
        for k, (w, b) in enumerate(net):
            h = h @ w.astype(dtype) + b.astype(dtype)
            if k < len(net) - 1:
                h = act(h)
        return h
