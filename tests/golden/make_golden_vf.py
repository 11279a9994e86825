"""Generate the golden vectors of the clipped value loss and the per-minibatch advantage normalisation by running the
UNMODIFIED reference with those two options added in torch fp32 around it.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_vf.py

The recipe is make_golden.py's run_fixture (3 steps on one minibatch, the first one clipped by the reference's
clip_policy_grad, torch.optim.Adam), on the seeds and states of the fixture of the same name without "_vf", through the
reference's value_net, ppo_entropy_loss, clip_policy_grad and Adam, with two changes:

  * the minibatch's advantages are normalised first, as Stable-Baselines3 does, over its graphs with exps != 0:
    (A - A[ind].mean()) / (A[ind].std() + 1e-8) in torch fp32, for every graph;
  * AgentPG.value_loss is replaced by the clipped value loss of OpenAI baselines' ppo2 / CleanRL's clip_vloss,
        mean(torch.max((V - R)^2, (V_old + torch.clamp(V - V_old, -c, c) - R)^2))
    with V_old = the values before the first step plus fixed per-graph offsets, chosen so that step 0 has all four
    cases of the seed: an exact tie (offset 0), inside the clamp, the clipped term larger, the unclipped term larger.

  * small_mixed_vf  SGNN, mixed stages, exps[1] = 0, value_clip 0.1;
  * mlp_small_vf    the rl-mlp model, value_clip 0.1.

Each file stores `advantages` (the raw inputs), `advantages_normalized` (what the reference was fed), `old_values`,
`value_clip` and `normalize_advantage`.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)
import torch  # noqa: E402

VALUE_CLIP = 0.1
FIXTURES = [
    # name, community, seed, count, rl-mlp
    ("small_mixed_vf", "small", 5, 8, False),
    ("mlp_small_vf", "small", 5, 12, True),
]


def offsets(v, r, c):
    """Per graph, by position mod 4: 0 (exact tie), +-0.4 c (inside the clamp), 2.5 c away from R (the clipped term
    larger), 1.3 c toward R (the unclipped term larger)."""
    s = np.where(v >= r, 1.0, -1.0)
    i = np.arange(v.size)
    out = np.select([i % 4 == 0, i % 4 == 1, i % 4 == 2],
                    [0.0, 0.4 * c * np.where((i // 4) % 2 == 0, 1.0, -1.0), 2.5 * c * s], -1.3 * c * s)
    return out.astype(np.float32)


def branches(v, r, v_old, c):
    d = v - v_old
    vc = v_old + torch.clamp(d, -c, c)
    a, b = (v - r).pow(2), (vc - r).pow(2)
    return {"tie": bool((a == b).any()), "inside": bool(((d.abs() < c) & (d != 0)).any()),
            "clipped": bool((b > a).any()), "unclipped": bool(((a > b) & (d.abs() > c)).any())}


def run(name, community, seed, count, mlp):
    from khrylib.rl.agents import AgentPG
    kept = {}

    def normalise(flat, states, actions, adv, ret, exps):
        a = torch.tensor(adv)
        ind = torch.tensor(exps).nonzero(as_tuple=False).squeeze(1)
        normed = (a - a[ind].mean()) / (a[ind].std() + 1e-8)
        kept["raw"], kept["normalized"] = adv, normed.numpy()
        return {"advantages": normed.numpy()}

    def clipped_value_loss(self, states, returns):
        values_pred = self.value_net(self.trans_value(states))
        if "old" not in kept:                      # step 0: the values before any step
            v0 = values_pred.detach().numpy().reshape(-1)
            r0 = returns.numpy().reshape(-1)
            old = (v0 + offsets(v0, r0, VALUE_CLIP)).astype(np.float32)
            kept["old"] = old.reshape(values_pred.shape)
            kept["branches"] = branches(values_pred.detach(), returns, torch.tensor(kept["old"]), VALUE_CLIP)
        old = torch.tensor(kept["old"])
        vc = old + torch.clamp(values_pred - old, -VALUE_CLIP, VALUE_CLIP)
        return torch.max((values_pred - returns).pow(2), (vc - returns).pow(2)).mean()

    ref = AgentPG.value_loss
    AgentPG.value_loss = clipped_value_loss
    try:
        MG.run_fixture(name, community, seed, count, mlp=mlp, case=normalise)
    finally:
        AgentPG.value_loss = ref
    assert all(kept["branches"].values()), kept["branches"]
    path = os.path.join(HERE, f"{name}.npz")
    z = dict(np.load(path))
    z.update(advantages=np.asarray(kept["raw"], np.float32), advantages_normalized=kept["normalized"].astype(np.float32),
             old_values=kept["old"].astype(np.float32), value_clip=np.float64(VALUE_CLIP),
             normalize_advantage=np.int64(1))
    np.savez_compressed(path, **z)


if __name__ == "__main__":
    only = set(sys.argv[1:])
    print("torch", torch.__version__, "reference at", MG.ref_shim.REFERENCE_ROOT)
    for fx in FIXTURES:
        if not only or fx[0] in only:
            run(*fx)
