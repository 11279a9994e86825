"""CPU: the uniforms InferenceServer hands to select_action stay inside the [0, 1) the sampler is defined on.  The
workers draw them in float64 and the server passes float32; every draw in [1 - 2^-25, 1) would round to exactly 1.0."""
import numpy as np

from drl_urban_planning_b200 import synth
from drl_urban_planning_b200.server import InferenceServer


class _Draws:
    """Stand-in for a worker's numpy generator: returns the given values in turn."""

    def __init__(self, values):
        self.values = list(values)

    def random(self):
        return self.values.pop(0)


def test_worker_uniforms_reach_the_sampler_below_one():
    spec = synth.COMMUNITIES["tiny"]
    states, _ = synth.make_states(8, "tiny", 1)
    draws = [1.0 - 2.0 ** -30, 1.0 - 2.0 ** -25, 1.0 - 2.0 ** -24, 0.5, 0.0, 1.0 - 2.0 ** -26]
    seen = []

    def infer(sts, uniforms):                     # records what the engine would be given
        seen.append(np.array(uniforms))
        return np.zeros(len(sts), np.int64)

    with InferenceServer(infer, spec.max_num_nodes, spec.max_num_edges, num_workers=1) as server:
        client = server.client(0)
        client._rng = _Draws(draws)
        for _ in draws:
            client.select_action([states[0]], mean_action=False)
        client._rng = _Draws([1.0 - 2.0 ** -30])
        client.select_action([states[0]], mean_action=True)
    assert server.error is None
    got = np.concatenate(seen)
    assert got.dtype == np.float32 and got.shape == (len(draws) + 1,)
    below_one = np.nextafter(np.float32(1), np.float32(0))
    assert (got[:-1] >= 0).all() and (got[:-1] < 1).all(), got
    # the largest float32 below 1 for every draw that rounds up to 1.0f; the others exactly as float32 rounds them
    assert got[:-1].tolist() == [below_one, below_one, below_one, 0.5, 0.0, below_one]
    assert np.isnan(got[-1])                      # a greedy request still carries the NaN flag
