"""On-device policy for `BaseRLAviary.rollout` (SURVEY.md 8f rank 1; reference caller: examples/learn.py:67-95, SB3's
`PPO('MlpPolicy', env)` whose `collect_rollouts` alternates policy.forward and env.step).

`MlpPolicy` holds the weights of an SB3-MlpPolicy-shaped actor (flatten -> 64 tanh -> 64 tanh -> linear mean, state-independent
`log_std`) and optionally the critic (same trunk shape, one output) as row-major `[in][out]` float32 CUDA tensors, plus
the layout the rollout kernel reads: every matrix split once into two float16 parts (`hi` = fp16(W), `lo` = fp16(2048 (W - hi));
the tensor-core products hi*hi + 2^-11 (hi*lo + lo*hi) with fp32 accumulation then reproduce fp32), stored in the order of the
mma B fragments (one 16-byte load per lane, k-step and 8 outputs), rows zero-padded to a multiple of 16 and last-layer columns to 8.  `rollout(policy=...)` then evaluates it inside the kernel every tick, from the observation
window in shared memory: no policy launch, no action tensor round trip.  `forward_torch` is the same network in plain PyTorch
fp32 (what a learner would run for the gradient step); the tests hold the kernel to a float64 restatement of it."""
import copy
import ctypes as C

import torch

from . import _native as N


class MlpPolicy:
    HIDDEN = 64

    def __init__(self, actor, log_std, critic=None, device=None):
        """actor / critic: three (weight [in, out], bias [out]) pairs each; log_std: [out_dim]."""
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())

        def prep(net, last):
            if net is None:
                return None
            if len(net) != 3:
                raise ValueError("the on-device policy is a 3-layer MLP (in -> 64 -> 64 -> out)")
            out = []
            for k, (w, b) in enumerate(net):
                w = torch.as_tensor(w, dtype=torch.float32).to(dev).contiguous()
                b = torch.as_tensor(b, dtype=torch.float32).to(dev).contiguous()
                if w.dim() != 2 or b.shape != (w.shape[1],):
                    raise ValueError("layer %d: weight must be [in, out] and bias [out]" % k)
                out.append((w, b))
            if out[0][0].shape[1] != self.HIDDEN or out[1][0].shape != (self.HIDDEN, self.HIDDEN) or out[2][0].shape[0] != self.HIDDEN:
                raise ValueError("hidden width must be 64 (SB3 MlpPolicy default)")
            if last is not None and out[2][0].shape[1] != last:
                raise ValueError("last layer must have %d outputs" % last)
            return out

        self.actor = prep(actor, None)
        self.in_dim, self.out_dim = self.actor[0][0].shape[0], self.actor[2][0].shape[1]
        self.critic = prep(critic, 1)
        if self.critic is not None and self.critic[0][0].shape[0] != self.in_dim:
            raise ValueError("critic input width differs from the actor's")
        self.log_std = torch.as_tensor(log_std, dtype=torch.float32).to(dev).contiguous().reshape(self.out_dim)
        self.device = dev
        if self.out_dim > 32:
            raise ValueError("the on-device policy supports up to 32 action outputs per aviary (D * A)")
        self.nt3 = 1 if self.out_dim <= 8 else (2 if self.out_dim <= 16 else 4)
        self._split = {"actor": self._prepare(self.actor, 8 * self.nt3), "critic": None if self.critic is None else self._prepare(self.critic, 8)}

    @staticmethod
    def _fragment_order(hi, lo, first_layer):
        """[Kpad, Npad] float16 parts -> [Kpad / 16, Npad / 8, 32, 4] int32: per (k-step, n-tile, lane) the lane's B-fragment
        registers of mma.m16n8k16 {b0 hi, b1 hi, b0 lo', b1 lo'} (include/quadsim.h, QsPolicy).  Lane = 4 g + t holds column 8 n + g
        and the k pairs (ka, ka + 1), (kb, kb + 1) with (ka, kb) = (2 t, 2 t + 8), or (4 t, 4 t + 2) for the first layer."""
        K, Nc = hi.shape
        dev = hi.device
        lane = torch.arange(32, device=dev)
        g, t = lane // 4, lane % 4
        ka, kb = (4 * t, 4 * t + 2) if first_layer else (2 * t, 2 * t + 8)
        ks = torch.arange(K // 16, device=dev).view(-1, 1, 1) * 16
        col = (torch.arange(Nc // 8, device=dev).view(1, -1, 1) * 8 + g.view(1, 1, -1)).expand(K // 16, -1, -1)

        def pair(part, k):                                   # {part[k][col], part[k + 1][col]} -> low half, high half
            u = part.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
            rows = (ks + k.view(1, 1, -1)).expand(-1, Nc // 8, -1)
            return u[rows, col] | (u[rows + 1, col] << 16)
        return torch.stack([pair(hi, ka), pair(hi, kb), pair(lo, ka), pair(lo, kb)], dim=-1).contiguous()

    def _prepare(self, net, last_cols):
        """[(fragment-ordered weights, bias)] x 3 with zero-padded rows (multiple of 16) and last-layer columns."""
        out = []
        for k, (w, b) in enumerate(net):
            rows = (w.shape[0] + 15) // 16 * 16
            cols = last_cols if k == 2 else w.shape[1]
            wp = torch.zeros((rows, cols), dtype=torch.float32, device=w.device)
            wp[:w.shape[0], :w.shape[1]] = w
            bp = torch.zeros((cols,), dtype=torch.float32, device=w.device)
            bp[:b.shape[0]] = b
            hi = wp.clamp(-65504.0, 65504.0).to(torch.float16)
            lo = ((wp - hi.to(torch.float32)) * 2048.0).clamp(-65504.0, 65504.0).to(torch.float16)
            out.append((self._fragment_order(hi, lo, k == 0), bp.contiguous()))
        return out

    @classmethod
    def from_linear(cls, actor_layers, log_std, critic_layers=None, device=None):
        """From torch.nn.Linear modules (weight [out, in]): e.g. SB3's mlp_extractor.policy_net[0], [2] and action_net."""
        t = lambda ls: None if ls is None else [(l.weight.detach().t().contiguous(), l.bias.detach()) for l in ls]   # noqa: E731
        return cls(t(actor_layers), log_std, t(critic_layers), device)

    @classmethod
    def random(cls, in_dim, out_dim, seed=0, critic=True, log_std=-0.5, device=None):
        g = torch.Generator().manual_seed(seed)

        def net(o):
            dims = [(in_dim, cls.HIDDEN), (cls.HIDDEN, cls.HIDDEN), (cls.HIDDEN, o)]
            return [((torch.rand(i, j, generator=g) * 2 - 1) / i ** 0.5, (torch.rand(j, generator=g) * 2 - 1) * 0.1) for i, j in dims]
        return cls(net(out_dim), torch.full((out_dim,), float(log_std)), net(1) if critic else None, device)

    # ---- the same network in PyTorch fp32 ---------------------------------------------------------------------------------
    @staticmethod
    def _mlp(net, x):
        h = torch.tanh(x @ net[0][0] + net[0][1])
        h = torch.tanh(h @ net[1][0] + net[1][1])
        return h @ net[2][0] + net[2][1]

    def forward_torch(self, obs, noise=None):
        """obs [E, D, obs_dim] (or [E, in_dim]) -> (raw action [E, out_dim], log-prob [E], value [E] or None), in the dtype of
        the weights (float32; `double()` gives a float64 copy)."""
        x = obs.reshape(obs.shape[0], -1).to(self.log_std.dtype)
        mean = self._mlp(self.actor, x)
        eps = torch.zeros_like(mean) if noise is None else noise.reshape(mean.shape).to(mean.dtype)
        raw = mean + torch.exp(self.log_std) * eps
        logp = (-0.5 * eps * eps - self.log_std - 0.91893853320467274).sum(dim=1)
        val = None if self.critic is None else self._mlp(self.critic, x)[:, 0]
        return raw, logp, val

    def double(self):
        """A copy whose `forward_torch` runs in float64 on the same (fp32-valued) weights; the packed kernel layout is shared."""
        c = copy.copy(self)
        f64 = lambda net: None if net is None else [(w.double(), b.double()) for w, b in net]   # noqa: E731
        c.actor, c.critic, c.log_std = f64(self.actor), f64(self.critic), self.log_std.double()
        return c

    # ---- C struct -------------------------------------------------------------------------------------------------------
    def c_struct(self, noise=None, logprob=None, values=None):
        q = N.QsPolicy()
        a = self._split["actor"]
        (q.w1, q.b1), (q.w2, q.b2), (q.w3, q.b3) = [(w.data_ptr(), b.data_ptr()) for w, b in a]
        q.log_std = self.log_std.data_ptr()
        if self.critic is not None:
            c = self._split["critic"]
            (q.vw1, q.vb1), (q.vw2, q.vb2), (q.vw3, q.vb3) = [(w.data_ptr(), b.data_ptr()) for w, b in c]
        q.nt3 = self.nt3
        q.noise = None if noise is None else noise.data_ptr()
        q.logprob = None if logprob is None else logprob.data_ptr()
        q.values = None if values is None else values.data_ptr()
        q.in_dim, q.out_dim = self.in_dim, self.out_dim
        return q


_ = C
