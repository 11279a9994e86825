"""The C-ABI entry points of both models (upb_* for the SGNN, upb_mlp_* for rl-mlp): what every per-model call does
with a null context, null required pointers and empty inputs, how many kernels a 0-graph step launches, the
optimiser-state round trip with its first-step clip latch, and the loss read-out.  Both models run the same host code
(csrc/upb200.cu), so every check is made for each of them.

The null-context checks need no GPU: they run wherever the library loads."""
import ctypes as C

import numpy as np
import pytest
import torch

from drl_urban_planning_b200 import _lib, params as PL, synth
from drl_urban_planning_b200.engine import Engine
from drl_urban_planning_b200.packing import pack_states

PREFIX = {"sgnn": "", "mlp": "mlp_"}
# entry points that take a context first and report a null one as UPB_ERR_ARG
CTX_CALLS = ("forward", "select_action", "ppo_grad", "apply", "ppo_step", "rearm_clip", "read_losses",
             "get_opt_state", "set_opt_state", "grad_norms")


def null_args(fn):
    """Zero / null for every argument after the context."""
    out = []
    for t in fn.argtypes[1:]:
        out.append(0 if t is C.c_int else 0.0 if t is C.c_float else None)
    return out


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
@pytest.mark.parametrize("call", CTX_CALLS)
def test_null_context_is_refused_and_named(call, model):
    L = _lib.lib()
    who = PREFIX[model] + call
    fn = getattr(L, "upb_" + who)
    assert fn(None, *null_args(fn)) == -1
    assert L.upb_last_error() == f"{who}: null context".encode()


@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_null_context_queries_return_zero(model):
    L = _lib.lib()
    assert getattr(L, f"upb_{PREFIX[model]}next_step_fused")(None) == 0
    assert L.upb_grid_size(None) == 0
    assert L.upb_launch_count(None) == 0


# ---------------------------------------------------------------------------------------------------------------- GPU
class Setup:
    def __init__(self, model, clip_mode=_lib.CLIP_REFERENCE):
        self.dev = torch.device("cuda", 0)
        self.count = 8
        states, actions = synth.make_states(7, "small", self.count)
        adv, ret, exps = synth.make_ppo_targets(7, self.count)
        fixed = np.full((self.count, 1), -3.0, np.float32)
        flat = PL.MLP.default_init(7) if model == "mlp" else PL.default_init(7)
        self.blob = pack_states(states).to(self.dev)
        self.eng = Engine(self.dev, self.blob.n_cap, self.blob.e_cap, model=model, clip_mode=clip_mode)
        self.params = torch.as_tensor(flat, device=self.dev).clone()
        self.arrays = [torch.as_tensor(x, device=self.dev) for x in (actions, adv, ret, fixed, exps)]
        self.fn = lambda name: getattr(_lib.lib(), self.eng._p + name)
        self.who = lambda name: (PREFIX[model] + name).encode()

    def step_args(self, count=None, **null):
        """Arguments of ppo_grad / ppo_step after the context; the names in `null` are passed as null pointers."""
        a = dict(blob=self.blob.dev_ptr(), ids=None, count=self.count if count is None else count,
                 params=self.params.data_ptr(), actions=self.arrays[0].data_ptr(), adv=self.arrays[1].data_ptr(),
                 ret=self.arrays[2].data_ptr(), fixed=self.arrays[3].data_ptr(), exps=self.arrays[4].data_ptr(),
                 inv_batch=1.0 / self.count, inv_ind=1.0 / self.count, grad=self.eng.new_grad_buffer().data_ptr(),
                 stream=self.eng._stream())
        a.update({k: None for k in null})
        return list(a.values())


def refused(s, name, args, who=None):
    before = s.eng.launches
    assert s.fn(name)(s.eng._ctx, *args) == -1, name
    assert _lib.lib().upb_last_error().startswith(s.who(who or name) + b": "), (name, _lib.lib().upb_last_error())
    assert s.eng.launches == before, name


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_null_required_pointer_is_refused_before_launching(model):
    s = Setup(model)
    ctx_args = lambda: (s.blob.dev_ptr(), None, s.count)
    out = torch.zeros(s.count, dtype=torch.float32, device=s.dev)
    idx = torch.zeros(s.count, dtype=torch.int32, device=s.dev)
    refused(s, "forward", [None, None, s.count, s.params.data_ptr(), None, out.data_ptr(), None, None, None, None])
    refused(s, "forward", [*ctx_args(), None, None, out.data_ptr(), None, None, None, None])
    refused(s, "forward", [s.blob.dev_ptr(), None, -1, s.params.data_ptr(), None, out.data_ptr(), None, None, None,
                           None])
    refused(s, "select_action", [*ctx_args(), s.params.data_ptr(), None, None, None])
    refused(s, "select_action", [*ctx_args(), None, None, idx.data_ptr(), None])
    for name in ("params", "actions", "adv", "ret", "fixed", "exps", "grad"):
        refused(s, "ppo_grad", s.step_args(**{name: None}))
    # the first step of CLIP_REFERENCE clips: ppo_step runs the two-call path, whose ppo_grad reports the error
    refused(s, "ppo_step", s.step_args(adv=None), who="ppo_grad")
    grad = s.eng.new_grad_buffer()
    refused(s, "apply", [None, grad.data_ptr(), None])
    refused(s, "apply", [s.params.data_ptr(), None, None])
    refused(s, "read_losses", [None, (C.c_float * 4)(), None])
    refused(s, "read_losses", [grad.data_ptr(), None, None])
    refused(s, "grad_norms", [None, 1, out.data_ptr(), None])
    refused(s, "grad_norms", [grad.data_ptr(), 1, None, None])
    refused(s, "grad_norms", [grad.data_ptr(), -1, out.data_ptr(), None])
    f = Setup(model, clip_mode=_lib.CLIP_NEVER)      # a fused step checks its own arguments
    assert f.eng.next_step_fused()
    for name in ("params", "actions", "adv", "ret", "fixed", "exps", "grad"):
        refused(f, "ppo_step", f.step_args(**{name: None}))
    torch.cuda.synchronize()
    assert s.eng.get_opt_state()[2].tolist() == f.eng.get_opt_state()[2].tolist() == [0, 0, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_empty_inputs_launch_as_documented(model):
    """count == 0: forward and select_action launch nothing; ppo_grad launches the reduction only (a zero gradient
    buffer, statistics included); ppo_step on one GPU takes the two-call path (reduction + Adam) in every clip mode."""
    for clip_mode in (_lib.CLIP_REFERENCE, _lib.CLIP_NEVER):
        s = Setup(model, clip_mode)
        out = torch.zeros(s.count, dtype=torch.float32, device=s.dev)
        idx = torch.zeros(s.count, dtype=torch.int32, device=s.dev)
        assert s.fn("forward")(s.eng._ctx, s.blob.dev_ptr(), None, 0, s.params.data_ptr(), None, out.data_ptr(),
                               None, None, None, None) == 0
        assert s.fn("select_action")(s.eng._ctx, s.blob.dev_ptr(), None, 0, s.params.data_ptr(), None,
                                     idx.data_ptr(), None) == 0
        assert s.eng.launches == 0
        grad = torch.full((s.eng.grad_stride,), float("nan"), dtype=torch.float32, device=s.dev)
        args = s.step_args(count=0)
        args[-2] = grad.data_ptr()
        assert s.fn("ppo_grad")(s.eng._ctx, *args) == 0
        assert s.eng.launches == 1
        torch.cuda.synchronize()
        assert not grad.cpu().numpy().any()
        p0 = s.params.cpu().numpy()
        assert s.fn("ppo_step")(s.eng._ctx, *s.step_args(count=0)) == 0
        assert s.eng.launches == 3
        torch.cuda.synchronize()
        assert np.array_equal(s.params.cpu().numpy(), p0)
        assert s.eng.get_opt_state()[2].tolist() == [1, 1, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["sgnn", "mlp"])
def test_opt_state_round_trip_and_first_step_clip(model):
    """set_opt_state -> get_opt_state returns the very bits; the restored global step arms the first-step clip when
    it is 0 and disarms it otherwise (CLIP_REFERENCE), which next_step_fused() shows.  The other model's state is
    untouched."""
    s = Setup(model)
    n = s.eng.num_params
    rng = np.random.default_rng(3)
    m = rng.standard_normal(n).astype(np.float32)
    v = np.abs(rng.standard_normal(n)).astype(np.float32)
    m[:4] = [-0.0, np.float32(1e-45), np.float32(-3.4e38), np.float32(1.17e-38)]
    assert not s.eng.next_step_fused()                                   # a new context clips its first step
    for steps, fused in (([5, 5, 3, 2], True), ([0, 0, 0, 0], False), ([1, 1, 1, 0], True)):
        s.eng.set_opt_state(m, v, np.array(steps, np.int64))
        assert s.eng.next_step_fused() == fused, steps
        m2, v2, st2 = s.eng.get_opt_state()
        assert m2.view(np.uint32).tolist() == m.view(np.uint32).tolist()
        assert v2.view(np.uint32).tolist() == v.view(np.uint32).tolist()
        assert st2.tolist() == steps
        m, v = v, m
    other = "sgnn" if model == "mlp" else "mlp"
    n_other = _lib.UPB_NUM_PARAMS if other == "sgnn" else _lib.UPB_MLP_NUM_PARAMS
    om, ov, ost = np.ones(n_other, np.float32), np.ones(n_other, np.float32), np.ones(4, np.int64)
    L = _lib.lib()
    assert getattr(L, f"upb_{PREFIX[other]}get_opt_state")(s.eng._ctx, om.ctypes.data, ov.ctypes.data,
                                                          ost.ctypes.data) == 0
    assert not om.any() and not ov.any() and ost.tolist() == [0, 0, 0, 0]
    assert getattr(L, f"upb_{PREFIX[other]}next_step_fused")(s.eng._ctx) == 0


@pytest.mark.gpu
def test_read_losses_is_the_same_for_both_models():
    """The four losses from the statistics block at each model's offset: identical numbers from identical blocks,
    the value loss over the sample count and the policy terms over the count of exps != 0 (1 when that is 0)."""
    dev = torch.device("cuda", 0)
    engines = {m: Engine(dev, 64, 128, model=m) for m in ("sgnn", "mlp")}
    rng = np.random.default_rng(5)
    for count_b, count_i in ((12.0, 7.0), (0.0, 0.0)):
        st = rng.standard_normal(_lib.UPB_STAT_COUNT).astype(np.float32)
        st[3], st[4] = count_b, count_i
        got = {}
        for name, eng in engines.items():
            g = eng.new_grad_buffer()
            g[eng.stat_offset:] = torch.as_tensor(st, device=dev)
            got[name] = eng.read_losses(g)
        assert got["sgnn"] == got["mlp"]
        f = np.float32
        value_loss, surr, ent = f(st[0] / f(max(count_b, 1))), f(st[1] / f(max(count_i, 1))), f(st[2] / f(max(count_i, 1)))
        expect = (surr + f(0.5) * value_loss + f(0.01) * ent, value_loss, surr, ent)
        assert np.allclose(got["sgnn"], expect, rtol=1e-6, atol=0), (got["sgnn"], expect)
