"""Record the masked policy logits of existing golden fixtures by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_logits.py [name ...]

For each fixture below, the states and flat parameters stored in `<name>.npz` (written by make_golden.py or
make_golden_extremes.py) are loaded into the reference model built by its own factory on the fixture's caps, and
`policy_net.forward` (urban_planning/models/policy.py:45-65) is run on the whole batch.  `<name>_logits.npz` then holds

  * lu_logits / lu_probs   (B0, max_num_edges): `logits` and `probs` of the land-use Categorical (absent if None),
  * rd_logits / rd_probs   (B1, max_num_nodes): the same of the road Categorical (absent if None),
  * stage                  (B, 3): the stage rows the reference returns.

`logits` are the reference's normalised logits (masked entries MASK_FILL - logsumexp, which rounds back to MASK_FILL
wherever a row has a candidate); edge_empty's all-masked rows normalise to 0 in fp32.  No new seeds: every input is
that of the existing fixture.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG  # noqa: E402  (installs the reference shim, sets up the paths)
import torch  # noqa: E402

from drl_urban_planning_b200 import params as PL  # noqa: E402
from fixtures_io import expand_states  # noqa: E402
from oracle import ref_shim  # noqa: E402

# name, rl-mlp
FIXTURES = [
    ("small_mixed", False),
    ("hlg", False),
    ("concept", False),
    ("edge_empty", False),
    ("extreme_heads", False),
    ("mlp_small", True),
    ("mlp_extreme_heads", True),
]


def record_logits(name, mlp):
    z = np.load(os.path.join(HERE, f"{name}.npz"))
    states = expand_states(z)
    build = ref_shim.build_reference_mlp_model if mlp else ref_shim.build_reference_model
    policy_net, _, ac = build(int(z["n_cap"]), int(z["e_cap"]), 111)
    L = PL.MLP if mlp else PL.SGNN
    ac.load_state_dict({k: torch.tensor(v) for k, v in L.to_state_dict(z["params"]).items()})
    with torch.no_grad():
        d0, d1, stage = policy_net(MG.tensorfy(states))
    out = dict(stage=stage.numpy().astype(np.float32),
               meta=np.array([f"torch {torch.__version__}", f"fixture {name}"]))
    for tag, d in (("lu", d0), ("rd", d1)):
        if d is not None:
            out[f"{tag}_logits"] = d.logits.numpy()
            out[f"{tag}_probs"] = d.probs.numpy()
    path = os.path.join(HERE, f"{name}_logits.npz")
    np.savez_compressed(path, **out)
    print(f"{name}: land use {None if d0 is None else tuple(d0.logits.shape)}, "
          f"road {None if d1 is None else tuple(d1.logits.shape)} -> {path} ({os.path.getsize(path) / 1024:.0f} KB)")


if __name__ == "__main__":
    only = set(sys.argv[1:])
    for name, mlp in FIXTURES:
        if not only or name in only:
            record_logits(name, mlp)
