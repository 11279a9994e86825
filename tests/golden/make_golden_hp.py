"""Generate the non-default-hyperparameter golden vectors in this directory by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_hp.py

The recipes are those of make_golden.py (run_fixture / run_update_params), on the same seeds and states as the fixture of
the same name without "_hp" / "_hp0", with the cfg's clip_epsilon, value_pred_coef, entropy_coef, lr, eps (and, for the
update, gamma / tau) set away from hlg.yaml's values.  Each file stores its settings under the same names.

  * small_mixed_hp   SGNN, mixed stages, 3 steps, the first one clipped: eps 0.18 (its fp32-formed clip bound 1.f + eps
                     is one ulp above torch.clamp's), c_v 1.0, c_e 0.05, lr 1e-3, Adam eps 1e-8;
  * small_mixed_hp0  SGNN with c_v = 0 and c_e = 0 (eps 0.33, whose fp32-formed lower bound is one ulp off): the value
                     head's parameters get a zero .grad, not None, so Adam still counts their steps.  The file records
                     that (value_grad_zero, value_adam_steps);
  * mlp_small_hp     the rl-mlp model: eps 0.18, c_v 0.25, c_e 0.05, lr 1e-3;
  * update_small_hp  the reference's whole update_params iteration with gamma 1.0, tau 0.0 (the shipped values;
                     update_small uses 0.99 / 0.95), eps 0.09, c_v 0.25, c_e 0.02, lr 3e-4.
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
    # name, community, seed, count, rl-mlp, settings
    ("small_mixed_hp", "small", 5, 8, False,
     dict(clip_epsilon=0.18, value_pred_coef=1.0, entropy_coef=0.05, lr=1e-3, eps=1e-8)),
    ("small_mixed_hp0", "small", 5, 8, False,
     dict(clip_epsilon=0.33, value_pred_coef=0.0, entropy_coef=0.0, lr=4e-4, eps=1e-5)),
    ("mlp_small_hp", "small", 5, 12, True,
     dict(clip_epsilon=0.18, value_pred_coef=0.25, entropy_coef=0.05, lr=1e-3, eps=1e-5)),
]
UPDATE = ("update_small_hp", dict(gamma=1.0, tau=0.0, clip_epsilon=0.09, value_pred_coef=0.25, entropy_coef=0.02,
                                  lr=3e-4, eps=1e-5))


def record(name, **extra):
    path = os.path.join(HERE, f"{name}.npz")
    z = dict(np.load(path))
    z.update({k: np.asarray(v) for k, v in extra.items()})
    np.savez_compressed(path, **z)


def run_watched(name, community, seed, count, mlp, hp):
    """run_fixture, keeping hold of the reference's modules and its Adam, to record what Adam did with the value head."""
    nets, opts = [], []
    build_sgnn, build_mlp, adam = MG.ref_shim.build_reference_model, MG.ref_shim.build_reference_mlp_model, torch.optim.Adam

    def keep(builder):
        def f(*a, **k):
            out = builder(*a, **k)
            nets.append(out)
            return out
        return f

    class WatchedAdam(adam):
        def __init__(self, params, **kw):
            super().__init__(params, **kw)
            opts.append(self)

    MG.ref_shim.build_reference_model, MG.ref_shim.build_reference_mlp_model = keep(build_sgnn), keep(build_mlp)
    torch.optim.Adam = WatchedAdam
    try:
        MG.run_fixture(name, community, seed, count, mlp=mlp, **hp)
    finally:
        MG.ref_shim.build_reference_model, MG.ref_shim.build_reference_mlp_model = build_sgnn, build_mlp
        torch.optim.Adam = adam
    (policy_net, value_net, _), = nets
    opt, = opts
    policy_ids = {id(p) for p in policy_net.parameters()}
    head = [p for p in value_net.parameters() if id(p) not in policy_ids]
    zero = all(p.grad is not None and not p.grad.any() for p in head)
    steps = [int(opt.state[p]["step"]) if p in opt.state else 0 for p in head]
    return zero, steps


if __name__ == "__main__":
    only = set(sys.argv[1:])
    print("torch", torch.__version__, "reference at", MG.ref_shim.REFERENCE_ROOT)
    for name, community, seed, count, mlp, hp in FIXTURES:
        if not only or name in only:
            zero, steps = run_watched(name, community, seed, count, mlp, hp)
            extra = dict(hp)
            if hp["value_pred_coef"] == 0.0:
                assert zero and steps == [3] * len(steps), (zero, steps)
                extra.update(value_grad_zero=zero, value_adam_steps=np.array(steps, np.int64))
            record(name, **extra)
    name, hp = UPDATE
    if not only or name in only:
        MG.run_update_params(name=name, **hp)
        record(name, **hp)
