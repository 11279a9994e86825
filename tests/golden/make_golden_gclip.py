"""Generate the golden vectors of the global gradient-norm clip (`max_grad_norm`) by running the UNMODIFIED reference
with its per-group clip replaced by torch's global one.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_gclip.py

The recipe is make_golden.py's run_fixture (3 steps on one minibatch, torch.optim.Adam), on the seeds and states of the
fixture of the same name without "_gclip", through the reference's value_net, ppo_entropy_loss and Adam, with one
change: AgentPPO.clip_policy_grad (two groups, max norm 1, agent_ppo.py:43-46) is replaced on every step by

    torch.nn.utils.clip_grad_norm_(actor_critic.parameters(), max_grad_norm)

over the model's parameters, the shared encoder counted once.  max_grad_norm is chosen below every step's norm, so all
three recorded steps clip (coef < 1).

  * small_mixed_gclip  SGNN, mixed stages, exps[1] = 0;
  * mlp_small_gclip    the rl-mlp model.

Each file stores `max_grad_norm` and `grad_norms`, the fp32 total norm torch's clip measured on each step (`grads`
stays the gradient before the clip, as in every fixture).
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)
import torch  # noqa: E402

FIXTURES = [
    # name, community, seed, count, rl-mlp, max_grad_norm
    ("small_mixed_gclip", "small", 5, 8, False, 0.05),
    ("mlp_small_gclip", "small", 5, 12, True, 0.05),
]


def run(name, community, seed, count, mlp, max_norm):
    from khrylib.rl.agents import AgentPPO
    norms = []

    def global_clip(self):
        seen = {}
        for p in list(self.policy_net.parameters()) + list(self.value_net.parameters()):
            seen.setdefault(id(p), p)                  # actor_critic.parameters(): the shared encoder once
        norms.append(float(torch.nn.utils.clip_grad_norm_(list(seen.values()), max_norm)))

    ref = AgentPPO.clip_policy_grad
    AgentPPO.clip_policy_grad = global_clip
    try:
        MG.run_fixture(name, community, seed, count, mlp=mlp)
    finally:
        AgentPPO.clip_policy_grad = ref
    assert len(norms) == 3 and all(n > max_norm for n in norms), (norms, max_norm)
    path = os.path.join(HERE, f"{name}.npz")
    z = dict(np.load(path))
    z.update(max_grad_norm=np.float64(max_norm), grad_norms=np.array(norms, np.float32))
    np.savez_compressed(path, **z)
    print(f"{name}: max_grad_norm {max_norm}, norms {norms}")


if __name__ == "__main__":
    only = set(sys.argv[1:])
    print("torch", torch.__version__, "reference at", MG.ref_shim.REFERENCE_ROOT)
    for fx in FIXTURES:
        if not only or fx[0] in only:
            run(*fx)
