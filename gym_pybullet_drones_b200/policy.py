"""On-device policy for `BaseRLAviary.rollout` (SURVEY.md 8f rank 1; reference caller: examples/learn.py:67-95, SB3's
`PPO('MlpPolicy', env)` whose `collect_rollouts` alternates policy.forward and env.step).

`MlpPolicy` holds the weights of an SB3-MlpPolicy-shaped actor (flatten -> hidden layers -> linear mean, state-independent
`log_std`) and optionally the critic (its own hidden layers, one output) as row-major `[in][out]` float32 CUDA tensors.  Any SB3
`net_arch` with 1 to 4 hidden layers of 1 to 256 units per network is accepted, with independent actor and critic shapes
(`net_arch=dict(pi=[...], vf=[...])`) and one activation for the whole policy, Tanh (SB3's default) or ReLU, after every hidden
layer.  Next to the weights it keeps the layout the rollout kernel reads: every matrix split once into two float16 parts
(`hi` = fp16(W), `lo` = fp16(2048 (W - hi)); the tensor-core products hi*hi + 2^-11 (hi*lo + lo*hi) with fp32 accumulation then
reproduce fp32), stored in the order of the mma B fragments (one 16-byte load per lane, k-step and 8 outputs), rows zero-padded to
a multiple of 16, hidden columns to a multiple of 64 and last-layer columns to 8.  `rollout(policy=...)` then evaluates it inside
the kernel every tick, from the observation window in shared memory: no policy launch, no action tensor round trip.  The SB3
default, [64, 64] Tanh, runs through qs_rollout's register-resident evaluator (QsPolicy); every other shape through
qs_rollout_mlp (QsMlpPolicy), which stages the hidden activations in shared memory.  `forward_torch` is the same network in plain
PyTorch fp32 (what a learner would run for the gradient step); the tests hold the kernel to a float64 restatement of it.  Larger
networks run as `forward_torch` + `step()` per tick."""
import copy
import io
import os
import zipfile

import torch

from . import _native as N

ACTIVATIONS = {"tanh": N.MLP_TANH, "relu": N.MLP_RELU}


def _arch(net_arch):
    """SB3 net_arch (a list for both networks, or dict(pi=, vf=)) -> (pi, vf) lists of hidden widths."""
    if net_arch is None:
        return [MlpPolicy.HIDDEN, MlpPolicy.HIDDEN], [MlpPolicy.HIDDEN, MlpPolicy.HIDDEN]
    if isinstance(net_arch, dict):
        if set(net_arch) - {"pi", "vf"}:
            raise ValueError("net_arch dict takes the keys 'pi' and 'vf' only (no shared trunk)")
        return list(net_arch.get("pi", [])), list(net_arch.get("vf", []))
    return list(net_arch), list(net_arch)


class MlpPolicy:
    HIDDEN = 64                  # SB3's default width (net_arch [64, 64])
    MAX_HIDDEN_LAYERS = N.MLP_MAX_HIDDEN
    MAX_WIDTH = N.MLP_MAX_WIDTH
    MAX_OUT = 32
    _LIMITS = ("; the on-device policy takes 1 to %d hidden layers of 1 to %d units, Tanh or ReLU, up to %d outputs: run larger "
               "networks as forward_torch + step() per tick" % (N.MLP_MAX_HIDDEN, N.MLP_MAX_WIDTH, 32))

    def __init__(self, actor, log_std, critic=None, device=None, activation="tanh"):
        """actor / critic: 2 to 5 (weight [in, out], bias [out]) pairs each (1 to 4 hidden layers and the output layer);
        log_std: [out_dim]; activation: "tanh" or "relu", after every hidden layer of both networks."""
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if activation not in ACTIVATIONS:
            raise ValueError("activation must be 'tanh' or 'relu', not %r" % (activation,) + self._LIMITS)
        self.activation = activation

        def prep(net, last, which):
            if net is None:
                return None
            net = list(net)
            if not 2 <= len(net) <= self.MAX_HIDDEN_LAYERS + 1:
                raise ValueError("%s: %d hidden layers" % (which, len(net) - 1) + self._LIMITS)
            out = []
            for k, (w, b) in enumerate(net):
                w = torch.as_tensor(w, dtype=torch.float32).to(dev).contiguous()
                b = torch.as_tensor(b, dtype=torch.float32).to(dev).contiguous()
                if w.dim() != 2 or b.shape != (w.shape[1],):
                    raise ValueError("%s layer %d: weight must be [in, out] and bias [out]" % (which, k))
                if k > 0 and w.shape[0] != out[-1][0].shape[1]:
                    raise ValueError("%s layer %d takes %d inputs, the layer before gives %d" % (which, k, w.shape[0], out[-1][0].shape[1]))
                if k < len(net) - 1 and not 1 <= w.shape[1] <= self.MAX_WIDTH:
                    raise ValueError("%s hidden layer %d is %d units wide" % (which, k, w.shape[1]) + self._LIMITS)
                out.append((w, b))
            if last is not None and out[-1][0].shape[1] != last:
                raise ValueError("%s: last layer must have %d outputs" % (which, last))
            return out

        self.actor = prep(actor, None, "actor")
        self.in_dim, self.out_dim = self.actor[0][0].shape[0], self.actor[-1][0].shape[1]
        self.critic = prep(critic, 1, "critic")
        if self.critic is not None and self.critic[0][0].shape[0] != self.in_dim:
            raise ValueError("critic input width differs from the actor's")
        self.log_std = torch.as_tensor(log_std, dtype=torch.float32).to(dev).contiguous().reshape(self.out_dim)
        self.device = dev
        if self.out_dim > self.MAX_OUT:
            raise ValueError("the on-device policy supports up to 32 action outputs per aviary (D * A)")
        self.nt3 = 1 if self.out_dim <= 8 else (2 if self.out_dim <= 16 else 4)
        hidden = lambda net: [w.shape[1] for w, _ in net[:-1]]   # noqa: E731
        self.net_arch = dict(pi=hidden(self.actor), vf=None if self.critic is None else hidden(self.critic))
        # SB3's default shape keeps qs_rollout's register-resident evaluator; everything else goes through qs_rollout_mlp
        self.classic = activation == "tanh" and all(a in (None, [self.HIDDEN, self.HIDDEN]) for a in self.net_arch.values())
        self._split = {"actor": self._prepare(self.actor, 8 * self.nt3), "critic": None if self.critic is None else self._prepare(self.critic, 8)}

    @property
    def max_width(self):
        """Widest padded hidden layer of the two networks (what qs_rollout_mlp stages in shared memory)."""
        return max(w.shape[-3] * 8 for net in self._split.values() if net is not None for w, _ in net[:-1])

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
        """[(fragment-ordered weights, bias)] per layer: the first layer's rows zero-padded to a multiple of 16, hidden columns
        (and so the next layer's rows) to a multiple of 64, the last layer's columns to `last_cols`."""
        out = []
        rows = (net[0][0].shape[0] + 15) // 16 * 16
        for k, (w, b) in enumerate(net):
            cols = last_cols if k == len(net) - 1 else (w.shape[1] + 63) // 64 * 64
            wp = torch.zeros((rows, cols), dtype=torch.float32, device=w.device)
            wp[:w.shape[0], :w.shape[1]] = w
            bp = torch.zeros((cols,), dtype=torch.float32, device=w.device)
            bp[:b.shape[0]] = b
            hi = wp.clamp(-65504.0, 65504.0).to(torch.float16)
            lo = ((wp - hi.to(torch.float32)) * 2048.0).clamp(-65504.0, 65504.0).to(torch.float16)
            out.append((self._fragment_order(hi, lo, k == 0), bp.contiguous()))
            rows = cols
        return out

    @classmethod
    def from_linear(cls, actor_layers, log_std, critic_layers=None, device=None, activation="tanh"):
        """From torch.nn.Linear modules (weight [out, in]): e.g. SB3's mlp_extractor.policy_net[0], [2], ... and action_net."""
        t = lambda ls: None if ls is None else [(l.weight.detach().t().contiguous(), l.bias.detach()) for l in ls]   # noqa: E731
        return cls(t(actor_layers), log_std, t(critic_layers), device, activation)

    @classmethod
    def from_sb3(cls, src, activation="tanh", device=None):
        """From a trained SB3 `ActorCriticPolicy` (PPO / A2C 'MlpPolicy'): `src` is its state dict or the path of the SB3 zip
        (e.g. learn.py's best_model.zip), whose `policy.pth` member is read with torch.load(weights_only=True).  The activation
        is an argument because SB3 pickles policy_kwargs in the zip's `data` member, which is not read here: pass the
        activation_fn the model was trained with ("tanh", SB3's default, or "relu").  Maps mlp_extractor.policy_net.{0,2,4,6},
        action_net and log_std to the actor, mlp_extractor.value_net.{0,2,4,6} and value_net to the critic; any other parameter
        (a shared trunk, gSDE, a feature extractor with weights) raises ValueError naming it."""
        if isinstance(src, (str, os.PathLike)):
            with zipfile.ZipFile(src) as z:
                sd = torch.load(io.BytesIO(z.read("policy.pth")), map_location="cpu", weights_only=True)
        else:
            sd = dict(src)
        layers = {"pi": {}, "vf": {}}
        head = {}
        for key, v in sd.items():
            parts = key.split(".")
            if len(parts) == 4 and parts[0] == "mlp_extractor" and parts[1] in ("policy_net", "value_net") and parts[2].isdigit() \
                    and parts[3] in ("weight", "bias"):
                layers["pi" if parts[1] == "policy_net" else "vf"].setdefault(int(parts[2]), {})[parts[3]] = v
            elif key in ("action_net.weight", "action_net.bias", "value_net.weight", "value_net.bias", "log_std"):
                head[key] = v
            else:
                raise ValueError("from_sb3: parameter %r is outside the SB3 MlpPolicy mapping (mlp_extractor.policy_net / value_net, "
                                 "action_net, value_net, log_std)" % key)

        def net(which, out_key):
            idx = sorted(layers[which])
            if idx != list(range(0, 2 * len(idx), 2)):
                raise ValueError("from_sb3: mlp_extractor.%s layers %s are not SB3's Linear / activation sequence 0, 2, 4, ..."
                                 % ("policy_net" if which == "pi" else "value_net", idx))
            out = []
            for i in idx:
                if set(layers[which][i]) != {"weight", "bias"}:
                    raise ValueError("from_sb3: layer %d of %s lacks its weight or bias" % (i, which))
                out.append((layers[which][i]["weight"].t().contiguous(), layers[which][i]["bias"]))
            if out_key + ".weight" not in head or out_key + ".bias" not in head:
                raise ValueError("from_sb3: %s.weight / %s.bias missing" % (out_key, out_key))
            return out + [(head[out_key + ".weight"].t().contiguous(), head[out_key + ".bias"])]

        if "log_std" not in head:
            raise ValueError("from_sb3: log_std missing (a squashed or gSDE policy is out of scope)")
        critic = net("vf", "value_net") if ("value_net.weight" in head or layers["vf"]) else None
        return cls(net("pi", "action_net"), head["log_std"], critic, device, activation)

    @classmethod
    def random(cls, in_dim, out_dim, seed=0, critic=True, log_std=-0.5, device=None, net_arch=None, activation="tanh"):
        """Random weights of an SB3-shaped policy; net_arch as SB3's (default [64, 64] for both networks)."""
        g = torch.Generator().manual_seed(seed)
        pi, vf = _arch(net_arch)

        def net(o, hidden):
            widths = [in_dim] + list(hidden) + [o]
            dims = list(zip(widths[:-1], widths[1:]))
            return [((torch.rand(i, j, generator=g) * 2 - 1) / i ** 0.5, (torch.rand(j, generator=g) * 2 - 1) * 0.1) for i, j in dims]
        return cls(net(out_dim, pi), torch.full((out_dim,), float(log_std)), net(1, vf) if critic else None, device, activation)

    # ---- the same network in PyTorch fp32 ---------------------------------------------------------------------------------
    def _mlp(self, net, x):
        act = torch.tanh if self.activation == "tanh" else torch.relu
        h = x
        for w, b in net[:-1]:
            h = act(h @ w + b)
        return h @ net[-1][0] + net[-1][1]

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

    # ---- float64 parameters of the actor (differentiable_rollout(policy=)) -------------------------------------------------
    def parameters64(self):
        """[W1, b1, ..., Wout, bout, log_std]: float64 CUDA copies of the actor's weights ([in, out]), biases and log_std as
        leaves that require grad: what `differentiable_rollout(policy=self, params=...)` differentiates and an optimiser
        updates.  The critic is not part of it."""
        out = [t.detach().double().clone().requires_grad_(True) for wb in self.actor for t in wb]
        return out + [self.log_std.detach().double().clone().requires_grad_(True)]

    def load_parameters(self, params):
        """Writes a `parameters64()`-shaped list back into the actor (rounded to the weights' dtype) and re-packs the fp16
        fragments `rollout(policy=self)` reads.  The critic is left alone."""
        params = list(params)
        if len(params) != 2 * len(self.actor) + 1:
            raise ValueError("load_parameters takes %d tensors (weight and bias per actor layer, then log_std), got %d"
                             % (2 * len(self.actor) + 1, len(params)))
        new = []
        for k, (w, b) in enumerate(self.actor):
            nw, nb = params[2 * k], params[2 * k + 1]
            if tuple(nw.shape) != tuple(w.shape) or tuple(nb.shape) != tuple(b.shape):
                raise ValueError("load_parameters: layer %d must be weight %s and bias %s" % (k, tuple(w.shape), tuple(b.shape)))
            new.append((nw.detach().to(device=w.device, dtype=w.dtype).contiguous().clone(),
                        nb.detach().to(device=b.device, dtype=b.dtype).contiguous().clone()))
        if tuple(params[-1].shape) != tuple(self.log_std.shape):
            raise ValueError("load_parameters: log_std must be %s" % (tuple(self.log_std.shape),))
        self.actor = new
        self.log_std = params[-1].detach().to(device=self.log_std.device, dtype=self.log_std.dtype).contiguous().clone()
        self._split = dict(self._split, actor=self._prepare(self.actor, 8 * self.nt3))

    # ---- C structs ------------------------------------------------------------------------------------------------------
    def c_struct(self, noise=None, logprob=None, values=None):
        """QsPolicy (qs_rollout): the [64, 64] Tanh network only."""
        if len(self._split["actor"]) != 3 or (self.critic is not None and len(self._split["critic"]) != 3) \
                or self.max_width != self.HIDDEN or self.activation != "tanh":
            raise ValueError("QsPolicy describes the [64, 64] Tanh network only: use mlp_struct (qs_rollout_mlp)")
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

    def mlp_struct(self, noise=None, logprob=None, values=None):
        """QsMlpPolicy (qs_rollout_mlp): any supported shape."""
        q = N.QsMlpPolicy()

        def fill(dst, split):
            dst.depth = len(split) - 1
            for k, (w, b) in enumerate(split):
                dst.w[k], dst.b[k] = w.data_ptr(), b.data_ptr()
                if k < dst.depth:
                    dst.width[k] = w.shape[1] * 8
            dst.out_tiles = split[-1][0].shape[1]
        fill(q.actor, self._split["actor"])
        if self.critic is not None:
            fill(q.critic, self._split["critic"])
        q.activation = ACTIVATIONS[self.activation]
        q.in_dim, q.out_dim = self.in_dim, self.out_dim
        q.log_std = self.log_std.data_ptr()
        q.noise = None if noise is None else noise.data_ptr()
        q.logprob = None if logprob is None else logprob.data_ptr()
        q.values = None if values is None else values.data_ptr()
        return q
