"""CPU: the rounding oracle of the bf16-tile build (tests/bf16_oracle.py) and what tells that build apart from the
parity build.

  * bf16_round equals torch's fp32 -> bfloat16 conversion bit for bit on every class of fp32 value, and keeps a NaN
    a NaN;
  * the oracle's tile hook at identity is the float64 oracle, bit for bit; with the bf16 rounding it moves exactly the
    tensors the tiles reach (bf16_oracle.TILE_TENSORS), by far more than the 1e-4 parity bar, and leaves every other
    tensor, the losses and the forward results bit-identical;
  * where cuobjdump is on PATH: the two libraries' SASS performs different arithmetic only in the kernels that run the
    SGNN backward (k_sgnn<true>, k_sgnn_gclip, k_sgnn_pg), one tensor-core pass for three there, so every other entry
    point of the bf16 build computes what the parity build computes."""
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest
import torch

import bf16_oracle as BO
from drl_urban_planning_b200 import params as PL, synth
from fixtures_io import expand_states
from harness import load, tensor_errors
from oracle import sgnn_numpy as ON

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "drl_urban_planning_b200", f) for f in ("libupb200.so", "libupb200_bf16.so")]
TILE_KERNELS = {"_ZN3upb6k_sgnnILb1EEEvNS_8StepArgsE", "_ZN3upb12k_sgnn_gclipENS_8StepArgsE",
                "_ZN3upb9k_sgnn_pgENS_8StepArgsE"}


def f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def torch_bf16_bits(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def test_bf16_round_matches_torch_on_every_class():
    rng = np.random.default_rng(0)
    top = rng.integers(0, 1 << 16, 4096, dtype=np.uint32) << 16
    finite = [
        rng.standard_normal(20000).astype(np.float32),
        (rng.standard_normal(4000) * 1e-39).astype(np.float32),                   # subnormals
        f32(rng.integers(1, 0x800000, 4000, dtype=np.uint32)),                      # every subnormal width
        f32(top[(top & 0x7f800000) != 0x7f800000] | 0x8000),                        # ties: even and odd upper halves
        f32(np.array([0x3f808000, 0x3f818000, 0xbf808000, 0xbf818000, 0x00008000, 0x00018000], np.uint32)),
        f32(np.array([0x7f7f7fff, 0x7f7f8000, 0x7f7fffff, 0xff7f8000, 0xff7fffff, 0x7f7f0000], np.uint32)),  # near max
        f32(np.array([0x7f800000, 0xff800000, 0, 0x80000000], np.uint32)),          # +-inf, +-0
    ]
    x = np.concatenate(finite)
    got = BO.bf16_round(x).view(np.uint32)
    assert not (got & 0xffff).any()
    want = torch_bf16_bits(x)
    bad = np.flatnonzero((got >> 16).astype(np.uint16) != want)
    assert bad.size == 0, [(hex(x.view(np.uint32)[i]), hex(got[i] >> 16), hex(want[i])) for i in bad[:8]]
    # the classes really occur: rounding up to inf, both tie directions
    assert np.isinf(BO.bf16_round(f32([0x7f7f8000, 0xff7fffff]))).all()
    assert BO.bf16_round(f32([0x3f808000, 0x3f818000])).view(np.uint32).tolist() == [0x3f800000, 0x3f820000]
    # NaNs of every sign and payload stay NaN (torch's own NaN bit pattern depends on its code path)
    nans = f32(np.array([0x7fffffff, 0xffffffff, 0x7f800001, 0xff800001, 0x7fc00000, 0xffc00000, 0x7fbfffff,
                         0x7f808000, 0x7f80ffff], np.uint32))
    assert np.isnan(BO.bf16_round(nans)).all() and np.isnan(torch.from_numpy(nans).to(torch.bfloat16).float()).all()
    assert (BO.bf16_round(nans).view(np.uint32) == 0x7fc00000).all()


def test_bf16_round_of_fp32_rounds_once():
    """The oracle rounds each operand once from fp32; rounding the TF32 head (cvt.rna) again would differ on ~6 % of
    normal values by one bf16 ulp.  The two must be told apart, or a test against this oracle cannot see the double
    rounding."""
    x = np.random.default_rng(1).standard_normal(200000).astype(np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    tf32 = (((u + 0x1000) & 0xffffe000).astype(np.uint32)).view(np.float32)          # round half away on 10 bits
    twice = BO.bf16_round(tf32).view(np.uint32)
    once = BO.bf16_round(x).view(np.uint32)
    assert np.array_equal(once >> 16, torch_bf16_bits(x).astype(np.uint32))
    frac = float((twice != once).mean())
    assert 0.04 < frac < 0.08, frac


def test_bf16_tile_is_exact_on_bf16_values():
    rng = np.random.default_rng(2)
    a = BO.bf16_round(rng.standard_normal((40, 24)).astype(np.float32)).astype(np.float64)
    b = BO.bf16_round(rng.standard_normal((24, 16)).astype(np.float32)).astype(np.float64)
    assert np.array_equal(BO.bf16_tile(a, b), a @ b)
    c = rng.standard_normal((40, 24))
    assert not np.array_equal(BO.bf16_tile(c, b), c @ b)


def fixture(golden_dir, name):
    z = load(golden_dir, name)
    if "digest" in z.files:
        states, _ = synth.make_states(int(z["seed"]), str(z["community"]), int(z["count"]))
    else:
        states = expand_states(z)
    return z, states


def oracle_args(z, states):
    return (z["params"], states, z["actions"], z["advantages"], z["returns"], z["fixed_log_probs"], z["exps"])


@pytest.mark.parametrize("name", ["small_mixed", "dhm256"])
def test_hook_at_identity_is_the_float64_oracle(name, golden_dir):
    z, states = fixture(golden_dir, name)
    want = ON.ppo_minibatch(*oracle_args(z, states))
    got = ON.ppo_minibatch(*oracle_args(z, states), tile=lambda a, b: a @ b)
    for k in ("grad", "value", "log_prob", "entropy"):
        assert np.array_equal(got[k], want[k]), k
    assert [got[k] for k in ("loss", "value_loss", "surr_loss", "entropy_loss")] == \
           [want[k] for k in ("loss", "value_loss", "surr_loss", "entropy_loss")]


@pytest.mark.parametrize("name", ["small_mixed", "dhm256"])
def test_bf16_tiles_move_only_the_tile_tensors(name, golden_dir):
    z, states = fixture(golden_dir, name)
    exact = ON.ppo_minibatch(*oracle_args(z, states))
    bf = BO.ppo_minibatch(*oracle_args(z, states))
    errs = tensor_errors(bf["grad"], exact["grad"])
    print(f"\n[bf16 oracle] {name}: " + ", ".join(f"{k} {errs[k]:.3g}" for k in BO.TILE_TENSORS))
    for s in PL.SLOTS.values():
        a, b = bf["grad"][s.offset:s.offset + s.size], exact["grad"][s.offset:s.offset + s.size]
        if s.name in BO.TILE_TENSORS:
            assert errs[s.name] > 1e-3, (s.name, errs[s.name])
        else:
            assert np.array_equal(a, b), s.name
    for k in ("value", "log_prob", "entropy", "loss", "value_loss", "surr_loss", "entropy_loss"):
        assert np.array_equal(bf[k], exact[k]), k


# ---- SASS of the two builds ------------------------------------------------------------------------------------------
# nvcc does not emit the same instructions twice: between compilations of one source, load vectorisation, register
# allocation and scheduling vary (k_mlp and k_sgnn included).  What a kernel computes does not: the count of each
# floating-point and tensor-core opcode per kernel is the same in every build of a source, so the builds are compared on
# those counts.
ARITH = re.compile(r"(FFMA|FADD|FMUL|FMNMX|FSETP|FSET|FSEL|FCHK|FRND|MUFU|HMMA|DFMA|DADD|DMUL|F2F|F2I|I2F)\b")


def arith_ops(path):
    """{mangled kernel name: Counter of its floating-point and tensor-core opcodes} from cuobjdump -sass."""
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            assert name not in kernels, name
            kernels[name] = Counter()
            continue
        text = re.sub(r"/\*.*?\*/", "", line).strip()
        text = re.sub(r"^@!?U?P\w+\s+", "", text)                 # predicate guard
        if name is not None and text and ARITH.match(text):
            kernels[name][text.split()[0].rstrip(";")] += 1
    return kernels


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump is not on PATH")
def test_only_the_sgnn_backward_kernels_differ_between_the_builds():
    """Every kernel but the three that run the SGNN backward performs the same arithmetic in both libraries, and those
    three issue one tensor-core instruction in the bf16 build for the parity build's three (3xTF32)."""
    for p in LIBS:
        assert os.path.exists(p), f"{p} is missing: build() makes both libraries"
    parity, bf16 = (arith_ops(p) for p in LIBS)
    assert set(parity) == set(bf16) and TILE_KERNELS < set(parity), sorted(set(parity) ^ set(bf16))
    differ = {k for k in parity if parity[k] != bf16[k]}
    assert differ == TILE_KERNELS, sorted(differ ^ TILE_KERNELS)
    for k in TILE_KERNELS:
        mma_p = sum(c for op, c in parity[k].items() if op.startswith("HMMA"))
        mma_b = sum(c for op, c in bf16[k].items() if op.startswith("HMMA"))
        assert mma_b > 0 and mma_p == 3 * mma_b, (k, mma_p, mma_b)
