"""Drop-in model objects with the reference's names, constructor signature, parameter names and checkpoint keys.

    create_sgnn_model(cfg, agent) -> (policy_net, value_net)          reference models/model.py:8-19
    ActorCritic(policy_net, value_net)                                reference models/model.py:36-47
    policy_net.select_action(x, mean_action) / get_log_prob_entropy(x, action) / forward(x)   policy.py:45-104
    value_net(x) -> (B, 1)                                            value.py:36-39

The modules own ordinary torch Parameters built from the same torch.nn layers in the same order as the reference
(so `torch.manual_seed(s)` gives bit-identical initial weights and `state_dict()` has the same 52 keys), which keeps
`torch.optim.Adam(actor_critic.parameters())`, `to_device`, `to_cpu`, checkpoint save/load working unchanged.

Two execution paths, chosen by where the parameters live:
  * CUDA: every call goes through libupb200.so (packed blob -> fused sm_90a kernel).  No autograd graph is built
    here -- the training step is `PPOUpdater.minibatch_step` (fwd+bwd+clip+Adam in CUDA); there is no eager fallback.
  * CPU: rollout-time inference (`select_action` inside forked sampling workers, reference
    urban_planning_agent.py:49-91; khrylib/rl/agents/agent.py:75-100) in plain PyTorch on the unpadded graph.  The
    rollouts stay on the CPU by design; this path never touches the CUDA library, so it is fork-safe.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import params as PL

MASK_FILL = -2.0 ** 32 + 1


def _check_specs(cfg):
    se, ps, vs = cfg.state_encoder_specs, cfg.policy_specs, cfg.value_specs
    ok = (list(se["state_encoder_hidden_size"]) == [64, 16] and se["gcn_node_dim"] == 16 and se["num_gcn_layers"] == 2
          and se["num_edge_fc_layers"] == 1 and se["num_attention_heads"] == 1
          and list(ps["policy_land_use_head_hidden_size"]) == [32, 1]
          and list(ps["policy_road_head_hidden_size"]) == [32, 1]
          and list(vs["value_head_hidden_size"]) == [32, 32, 1])
    if not ok:
        raise NotImplementedError(
            "the sm_90a kernels are specialised for the shapes of every shipped cfg (state_encoder [64,16], "
            "gcn_node_dim 16, 2 GCN layers, 1 edge-fc layer, 1 attention head, heads [32,1], value [32,32,1])")


def _seq(pairs):
    s = nn.Sequential()
    for name, mod in pairs:
        s.add_module(name, mod)
    return s


class SGNNStateEncoder(nn.Module):
    """Parameter container + CPU forward of the shared state encoder (reference models/state_encoder.py:7-214)."""

    def __init__(self, cfg, agent):
        super().__init__()
        self.cfg, self.agent = cfg, agent
        if agent.node_dim != PL.NODE_DIM or agent.numerical_feature_size != PL.NUMERICAL_DIM:
            raise NotImplementedError("node_dim must be 23 and numerical_feature_size 52")
        d = cfg["gcn_node_dim"]
        self.numerical_feature_encoder = _seq([
            ("flatten_0", nn.Flatten()), ("linear_0", nn.Linear(PL.NUMERICAL_DIM, 64)), ("tanh_0", nn.Tanh()),
            ("linear_1", nn.Linear(64, 16)), ("tanh_1", nn.Tanh())])
        self.node_encoder = nn.Linear(agent.node_dim, d)
        self.edge_fc_layers = nn.ModuleList(
            [_seq([("linear_0", nn.Linear(2 * d, d)), ("tanh_0", nn.Tanh())]) for _ in range(cfg["num_gcn_layers"])])
        self.max_num_nodes, self.max_num_edges = cfg["max_num_nodes"], cfg["max_num_edges"]
        self.attention_layer = nn.MultiheadAttention(d, cfg["num_attention_heads"])
        self.attention_query_layer = nn.Linear(d, d)
        self.attention_key_layer = nn.Linear(d, d)
        self.attention_value_layer = nn.Linear(d, d)
        self.output_policy_land_use_size = d * 4
        self.output_policy_road_size = d
        self.output_value_size = d * 3 + cfg["state_encoder_hidden_size"][-1] + 3

    # CPU rollout path: one unpadded graph, plain torch.  Returns (he_last (e,16), h (n,16), hc (16,), sv (67,))
    def encode_one(self, state):
        numerical, nf, ei, cur, nmask, emask, _, _, stage = state
        n, e = int(nmask.sum()), int(emask.sum())
        x, edges = nf[:n], ei[:e]
        u, v = edges[:, 0], edges[:, 1]
        h_num = self.numerical_feature_encoder(numerical.reshape(1, -1))[0]
        h = self.node_encoder(x)
        hc = self.node_encoder(cur)
        deg = torch.bincount(torch.cat([u, v]), minlength=n).to(h.dtype)
        inv = 1.0 / (deg + 1e-6)
        he = h.new_zeros(e, h.shape[1])
        for layer in self.edge_fc_layers:
            lin = layer.linear_0
            d = h.shape[1]
            p = F.linear(h, lin.weight[:, :d], lin.bias)
            qq = F.linear(h, lin.weight[:, d:])
            he = 0.5 * (torch.tanh(p[u] + qq[v]) + torch.tanh(p[v] + qq[u]))
            agg = torch.zeros_like(h).index_add_(0, u, he).index_add_(0, v, he)
            h = h + agg * inv[:, None]
        m_e = he.mean(0) if e > 0 else h.new_full((h.shape[1],), float("nan"))
        att = self._attend(hc, h)
        sv = torch.cat([h_num, h.mean(0), m_e, att, stage.to(h.dtype)])
        return he, h, hc, sv

    def _attend(self, hc, h):
        d = h.shape[1]
        wi, bi = self.attention_layer.in_proj_weight, self.attention_layer.in_proj_bias
        q = F.linear(self.attention_query_layer(hc), wi[:d], bi[:d])
        k = F.linear(self.attention_key_layer(h), wi[d:2 * d], bi[d:2 * d])
        v = F.linear(self.attention_value_layer(h), wi[2 * d:], bi[2 * d:])
        a = torch.softmax(k @ q / (d ** 0.5), dim=0)
        return self.attention_layer.out_proj(a @ v)


def _states_on_cuda(x) -> bool:
    t = x[0][0]
    return isinstance(t, torch.Tensor) and t.is_cuda


class _EngineMixin:
    """CUDA dispatch shared by the policy and value modules: flat parameter snapshot + engine + packing."""

    def _layout(self):
        return PL.MLP if getattr(self.shared_net, "model_kind", "sgnn") == "mlp" else PL.SGNN

    def _flat_params(self, device):
        named = {}
        sn = dict(self.shared_net.named_parameters())
        own = dict(self.named_parameters())
        slots = self._layout().slots
        for s in slots.values():
            if s.owner == "enc":
                named[s.name] = sn[s.key]
            elif s.key in own:
                named[s.name] = own[s.key]
            else:
                named[s.name] = getattr(self, "_peer_params")()[s.key]
        return torch.cat([named[s.name].detach().reshape(-1).to(device, torch.float32) for s in slots.values()])

    def _engine(self, device):
        from .engine import Engine
        eng = getattr(self.shared_net, "_upb_engine", None)
        if eng is None or eng.device != torch.device(device):
            eng = Engine(device, self.shared_net.max_num_nodes, self.shared_net.max_num_edges,
                         model=getattr(self.shared_net, "model_kind", "sgnn"))
            self.shared_net._upb_engine = eng
        return eng

    def _cuda_forward(self, x, actions=None, want_greedy=False):
        from .packing import pack_states
        device = next(self.parameters()).device
        eng = self._engine(device)
        blob = pack_states(x, self.shared_net.max_num_nodes, self.shared_net.max_num_edges).to(device)
        return eng.forward(blob, self._flat_params(device), actions, want_greedy=want_greedy)

    def _cuda_sample(self, x, uniforms=None):
        from .packing import pack_states
        device = next(self.parameters()).device
        eng = self._engine(device)
        blob = pack_states(x, self.shared_net.max_num_nodes, self.shared_net.max_num_edges).to(device)
        if uniforms is None:
            uniforms = torch.rand(len(x), device=device)
        return eng.select_action(blob, self._flat_params(device), uniforms=uniforms)


class UrbanPlanningPolicy(nn.Module, _EngineMixin):
    """reference models/policy.py:5-104."""

    def __init__(self, cfg, agent, shared_net):
        super().__init__()
        self.cfg, self.agent, self.shared_net = cfg, agent, shared_net
        self.policy_land_use_head = _seq([
            ("land_use_linear_0", nn.Linear(shared_net.output_policy_land_use_size, 32)), ("land_use_tanh_0", nn.Tanh()),
            ("land_use_linear_1", nn.Linear(32, 1, bias=False)), ("land_use_flatten_1", nn.Flatten())])
        self.policy_road_head = _seq([
            ("road_linear_0", nn.Linear(shared_net.output_policy_road_size, 32)), ("road_tanh_0", nn.Tanh()),
            ("road_linear_1", nn.Linear(32, 1, bias=False)), ("road_flatten_1", nn.Flatten())])
        self._peer_params = lambda: {}

    # ---- CPU: masked logits over the padded width for one state (policy.py:48-61)
    def _logits_one(self, state):
        he, h, hc, _ = self.shared_net.encode_one(state)
        stage = state[8]
        if stage[0] > 0:
            feat = torch.cat([he, hc.expand_as(he), he * hc, he - hc], dim=1)
            z = self.policy_land_use_head(feat).reshape(-1)
            mask, width = state[6], self.shared_net.max_num_edges
        else:
            z = self.policy_road_head(h).reshape(-1)
            mask, width = state[7], self.shared_net.max_num_nodes
        full = z.new_full((width,), MASK_FILL)
        full[:z.numel()] = z
        return torch.where(mask.bool(), full, z.new_full((width,), MASK_FILL)), int(stage[:2].argmax())

    def forward(self, x):
        """(land_use_dist, road_dist, stage) like the reference: Categorical distributions over the masked logits of the
        land-use graphs (B0, max_num_edges) and of the road graphs (B1, max_num_nodes), in batch order, None for a stage
        without a graph, and the (B, 3) stage rows.  On CUDA the logits come from the fused forward kernel
        (upb_policy_logits) and carry no autograd graph, like value_net's output there."""
        if next(self.parameters()).is_cuda:
            from .packing import pack_states
            device = next(self.parameters()).device
            blob = pack_states(x, self.shared_net.max_num_nodes, self.shared_net.max_num_edges).to(device)
            lu, rd, _ = self._engine(device).policy_logits(blob, self._flat_params(device))
            stage = torch.stack([torch.as_tensor(s[8]) for s in x]).to(device, self.agent.dtype)
            d0 = torch.distributions.Categorical(logits=lu) if lu is not None else None
            d1 = torch.distributions.Categorical(logits=rd) if rd is not None else None
            return d0, d1, stage
        if _states_on_cuda(x):
            raise RuntimeError("states on CUDA need the modules on CUDA (policy_net.to(device))")
        stage = torch.stack([s[8] for s in x])
        rows = [self._logits_one(s) for s in x]
        lu = [r for r, sid in rows if sid == 0]
        rd = [r for r, sid in rows if sid == 1]
        d0 = torch.distributions.Categorical(logits=torch.stack(lu)) if lu else None
        d1 = torch.distributions.Categorical(logits=torch.stack(rd)) if rd else None
        return d0, d1, stage

    def select_action(self, x, mean_action=False, uniforms=None):
        """(B, 2) float32: column 0 land-use edge index, column 1 road node index (policy.py:67-85).
        On CUDA a batch of states is evaluated by the fused forward kernel: greedy arg-max (bit-exact), or, for
        mean_action=False, inverse-CDF sampling from `uniforms` (B values in [0,1); torch.rand on the device if None)."""
        if next(self.parameters()).is_cuda:
            if mean_action:
                _, _, _, greedy = self._cuda_forward(x, want_greedy=True)
            else:
                greedy = self._cuda_sample(x, uniforms)
            stage = np.stack([np.asarray(s[8].detach().cpu() if hasattr(s[8], "detach") else s[8]) for s in x])
            out = torch.zeros(len(x), 2, dtype=self.agent.dtype, device=greedy.device)
            sid = torch.as_tensor(stage[:, :2].argmax(1), device=greedy.device)
            out[torch.arange(len(x), device=greedy.device), sid] = greedy.to(self.agent.dtype)
            return out
        d0, d1, stage = self.forward(x)
        action = torch.zeros(stage.shape[0], 2, dtype=self.agent.dtype)
        if d0 is not None:
            a = d0.probs.argmax(dim=1) if mean_action else d0.sample()
            action[stage[:, 0].bool(), 0] = a.to(self.agent.dtype)
        if d1 is not None:
            a = d1.probs.argmax(dim=1) if mean_action else d1.sample()
            action[stage[:, 1].bool(), 1] = a.to(self.agent.dtype)
        return action

    def get_log_prob_entropy(self, x, action):
        """((B,1), (B,1)) -- policy.py:87-104."""
        if next(self.parameters()).is_cuda:
            _, lp, ent = self._cuda_forward(x, actions=action)
            return lp.unsqueeze(1), ent.unsqueeze(1)
        d0, d1, stage = self.forward(x)
        lp = torch.zeros(stage.shape[0], dtype=self.agent.dtype)
        ent = torch.zeros_like(lp)
        if d0 is not None:
            sel = stage[:, 0].bool()
            lp[sel] = d0.log_prob(action[sel, 0]); ent[sel] = d0.entropy()
        if d1 is not None:
            sel = stage[:, 1].bool()
            lp[sel] = d1.log_prob(action[sel, 1]); ent[sel] = d1.entropy()
        return lp.unsqueeze(1), ent.unsqueeze(1)


class UrbanPlanningValue(nn.Module, _EngineMixin):
    """reference models/value.py:4-39."""

    def __init__(self, cfg, agent, shared_net):
        super().__init__()
        self.cfg, self.agent, self.shared_net = cfg, agent, shared_net
        self.value_head = _seq([
            ("linear_0", nn.Linear(shared_net.output_value_size, 32)), ("tanh_0", nn.Tanh()),
            ("linear_1", nn.Linear(32, 32)), ("tanh_1", nn.Tanh()), ("linear_2", nn.Linear(32, 1))])
        self._peer_params = lambda: {}

    def forward(self, x):
        if next(self.parameters()).is_cuda:
            value, _, _ = self._cuda_forward(x)
            return value.unsqueeze(1)
        return torch.stack([self.value_head(self.shared_net.encode_one(s)[3]) for s in x])


def create_sgnn_model(cfg, agent):
    """reference models/model.py:8-19 (same construction order -> same seeded initialisation)."""
    _check_specs(cfg)
    shared_net = SGNNStateEncoder(cfg.state_encoder_specs, agent)
    policy_net = UrbanPlanningPolicy(cfg.policy_specs, agent, shared_net)
    value_net = UrbanPlanningValue(cfg.value_specs, agent, shared_net)
    # each module can assemble the full flat vector (the CUDA kernel evaluates both heads in one pass)
    policy_net._peer_params = lambda: dict(value_net.named_parameters())
    value_net._peer_params = lambda: dict(policy_net.named_parameters())
    return policy_net, value_net


class ActorCritic(nn.Module):
    """reference models/model.py:36-47."""

    def __init__(self, actor_net, value_net):
        super().__init__()
        self.actor_net = actor_net
        self.value_net = value_net

    def flat_parameters(self) -> np.ndarray:
        return PL.from_state_dict(self.state_dict())

    def load_flat_parameters(self, flat) -> None:
        sd = PL.to_state_dict(np.asarray(flat, dtype=np.float32))
        self.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
