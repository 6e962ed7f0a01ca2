"""The ping-pong schedule of the persistent wgmma contraction (anyedit_b200/csrc/gemm_wgmma.cu): each consumer warpgroup owns
whole 128 x BN units and runs its epilogue under the other warpgroup's products.  It changes the order in which tiles are
computed, never the arithmetic of one element, so every case of tests/test_gpu_contraction.py, forced through
ANYSD_GEMM_SCHED=pingpong at BN 64 and 128, must meet the same float64 bound and write exactly the bits (outputs, GroupNorm
and LayerNorm statistics) of the cooperative schedule.  Extra cases cover the unit counts the schedule is sensitive to: an odd
number of units per CTA, a CTA with a single unit (the second warpgroup has nothing to do), and many more k-blocks per unit
than operand-ring stages.

The schedule switch is read once per process, so every setting runs in a child process (this file with ``--worker``)."""
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_contraction as tc  # noqa: E402

pytestmark = pytest.mark.gpu

EXTRA = [
    # 139 row tiles: 139 units at BN 128 (one or two per CTA), 278 at BN 64 (two or three)
    tc._dense("pp_units_odd", 139 * 128 - 40, 128, 320, rpb=200, rowadd=True, res=True),
    # one unit in all: one CTA, whose second warpgroup gets none
    tc._dense("pp_single_unit", 96, 64, 200, rpb=96, rowadd=True, res=True, stats=True),
    # 41 k-blocks per unit against a ring of at most 6 stages
    tc._dense("pp_long_k", 1000, 448, 41 * 64 - 56, act=1, rpb=200, rowadd=True, res=True),
]
ALL = tc.ALL + EXTRA
CASES = {c["name"]: c for c in ALL}
assert len(CASES) == len(ALL)
NAMES = [c["name"] for c in ALL]


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    inputs = {c["name"]: tc._make_inputs(c, 2000 + i) for i, c in enumerate(ALL)}
    d = tmp_path_factory.mktemp("pingpong")
    torch.save(inputs, d / "inputs.pt")
    refs = {}

    def ref(name):
        if name not in refs:
            refs[name] = tc._reference(CASES[name], inputs[name])
        return refs[name]
    return SimpleNamespace(inputs=inputs, dir=d, ref=ref)


def _child(data, tag, env):
    out = data.dir / f"out_{tag}.pt"
    e = {k: v for k, v in os.environ.items() if not k.startswith("ANYSD_GEMM")}
    e.update(env)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker",
           str(data.dir / "inputs.pt"), str(out)]
    r = subprocess.run(cmd, env=e, cwd=tc.ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker {tag} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return torch.load(out)


def _check_all(data, got, label, same):
    failures = []
    for name in NAMES:
        try:
            worst = f"{tc._check(CASES[name], data.inputs[name], data.ref(name), got[name], label):.3f}"
        except AssertionError as e:
            worst = "FAIL"
            failures.append(str(e).splitlines()[0])
        print(f"{label:12s} {name:24s} worst err/bound {worst:6s} bit-identical to cooperative: {same[name]}")
    return failures


@pytest.fixture(scope="module")
def coop(data):
    return _child(data, "coop", {"ANYSD_GEMM_SCHED": "coop"})


@pytest.mark.parametrize("bn", (64, 128))
def test_pingpong_against_fp64_and_bit_identical_to_cooperative(data, coop, bn):
    got = _child(data, f"pp{bn}", {"ANYSD_GEMM_SCHED": "pingpong", "ANYSD_GEMM_BN": str(bn)})
    same = {n: tc._same_bits(got[n], coop[n]) for n in NAMES}
    failures = _check_all(data, got, f"pingpong{bn}", same)
    assert not failures, "\n".join(failures)
    assert not any(got[n]["split"] for n in NAMES), "a case expected to run unsplit ran split-K"
    differ = [n for n in NAMES if not same[n]]
    assert not differ, f"ping-pong BN={bn}: not bit-identical to the cooperative schedule: {differ}"


def test_cooperative_against_fp64(data, coop):
    """The extra cases under the cooperative schedule meet the bound too (the reference the ping-pong bits are held to)."""
    failures = []
    for c in EXTRA:
        try:
            tc._check(c, data.inputs[c["name"]], data.ref(c["name"]), coop[c["name"]], "coop")
        except AssertionError as e:
            failures.append(str(e).splitlines()[0])
    assert not failures, "\n".join(failures)


def _worker(argv):
    inp, outp = argv[0], argv[1]
    if tc.ROOT not in sys.path:
        sys.path.insert(0, tc.ROOT)
    from anyedit_b200 import ops
    inputs = torch.load(inp)
    torch.save(tc._run_cases(ops, [CASES[n] for n in NAMES], inputs), outp)
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["--worker"]:
    sys.exit(_worker(sys.argv[2:]))
