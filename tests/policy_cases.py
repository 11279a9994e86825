"""Policy-head cases shared by the action-selection and policy-logits tests: one graph with exactly k candidates at the
limits of the sampler's scan (tests/test_gpu_select.py), the float64 candidate logits of both models, and the
distributions the unmodified reference recorded for UrbanPlanningPolicy.forward (tests/golden/*_logits.npz)."""
import os

import numpy as np
import torch

import shape_cases as SC
from drl_urban_planning_b200 import params as PL, synth
from drl_urban_planning_b200.model import MASK_FILL, ActorCritic
from fixtures_io import expand_states
from harness import Agent, Cfg
from oracle import mlp_port as MP
from oracle import sgnn_numpy as ON

TOL = 1e-4
SEED = 17
KS = [1, 2, 31, 32, 33, 64, 65, 160, 161]
SPEC = synth.CommunitySpec("select", 200, 600, 20, 120, 4.0, 0.3)      # small caps: thousands of copies stay cheap
# logits fixture -> rl-mlp
LOGIT_FIXTURES = {"small_mixed": False, "hlg": False, "concept": False, "edge_empty": False, "extreme_heads": False,
                  "mlp_small": True, "mlp_extreme_heads": True}


def make_case(rng, k, stage, spec=SPEC):
    """A graph with exactly k candidates for `stage`, on the smallest node / edge counts that hold them."""
    if stage == 0:
        n, e = (60, 200) if k <= 200 else (1000, 3000)
    else:
        n, e = max(40, k + 9), max(40, k + 9)
    st, _ = synth.make_exact_state(rng, spec, n, e, k, stage)
    return st


def cases():
    """(label, state, stage): every k of KS for both stages, then an empty mask for each stage."""
    rng = np.random.default_rng(SEED)
    out = [(f"{'lu' if s == 0 else 'road'}_k{k}", make_case(rng, k, s), s) for s in (0, 1) for k in KS]
    out += [(f"{'lu' if s == 0 else 'road'}_empty", make_case(rng, 0, s), s) for s in (0, 1)]
    return out


def caps_case():
    st, _ = synth.make_exact_state(np.random.default_rng(SEED + 1), SC.SPEC, 1000, 3000, 3000, 0)
    return st


def flat_params(model, seed=SEED):
    return PL.default_init(seed) if model == "sgnn" else PL.MLP.default_init(seed)


def ref_logits(model, flat, st):
    """(idx, z): the candidates in index order (the kernel's scan order) and their float64 logits."""
    stage = int(np.argmax(st[8][:2]))
    if model == "sgnn":
        P = ON._p64(flat)
        c = ON.forward(P, ON.unpad(st), keep=True)["cache"]
        w1 = P["lu_w1" if stage == 0 else "road_w1"].reshape(-1)
        return c["idx"], (c["th"] @ w1 if c["idx"].size else np.zeros(0))
    P = MP.params_from_flat(flat, torch.float64)
    with torch.no_grad():
        zl, zr = MP.masked_logits(P, MP.stack_states([st]))
    idx = np.flatnonzero(st[6] if stage == 0 else st[7])
    return idx, (zl if stage == 0 else zr)[0].numpy()[idx]


def load_policy(name, golden_dir):
    """(fixture, recorded logits, the fixture's states, policy_net holding the fixture's parameters on the CPU)."""
    from drl_urban_planning_b200.mlp import create_mlp_model
    from drl_urban_planning_b200.model import create_sgnn_model
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    ref = np.load(os.path.join(golden_dir, name + "_logits.npz"))
    mlp = LOGIT_FIXTURES[name]
    policy_net, value_net = (create_mlp_model if mlp else create_sgnn_model)(Cfg(int(z["n_cap"]), int(z["e_cap"])),
                                                                          Agent())
    sd = (PL.MLP if mlp else PL.SGNN).to_state_dict(np.asarray(z["params"], np.float32))
    ActorCritic(policy_net, value_net).load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()})
    return z, ref, expand_states(z), policy_net


def check_distribution(tag, d, ref):
    """d: a Categorical (or None) against the recorded `<tag>_logits` / `<tag>_probs` (absent when the reference's was
    None): shape, masked entries bit for bit, candidates at the per-tensor bar."""
    if f"{tag}_logits" not in ref:
        assert d is None, tag
        return
    want_z, want_p = ref[f"{tag}_logits"], ref[f"{tag}_probs"]
    z, p = d.logits.detach().cpu().numpy(), d.probs.detach().cpu().numpy()
    assert z.shape == want_z.shape and p.shape == want_p.shape, (tag, z.shape, want_z.shape)
    masked = (want_z == np.float32(MASK_FILL)) | np.all(want_z == 0.0, axis=1, keepdims=True)
    assert np.array_equal(z[masked], want_z[masked]) and np.array_equal(p[masked], want_p[masked]), tag
    cand = ~masked
    if cand.any():
        dz = np.abs(z[cand].astype(np.float64) - want_z[cand]).max() / np.abs(want_z[cand]).max()
        assert dz < TOL, (tag, "logits", dz)
    dp = np.abs(p.astype(np.float64) - want_p).max() / np.abs(want_p).max()
    assert dp < TOL, (tag, "probs", dp)
