"""Cold-L2 repetitions of the MLP training step (tools/stress_chain.py): every repetition must reproduce the first one
bit-exactly in the forward outputs and to the rounding of the float atomics in the gradients.  A race between the
shared-memory operand stores and the asynchronous tensor-core reads of the GEMM kernels shows up here as a repetition
that differs."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_cold_l2_repetitions_are_reproducible(monkeypatch, capsys):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import stress_chain
    monkeypatch.setattr(sys, "argv", ["stress_chain.py", "40"])
    stress_chain.main()
    assert "stress ok: 40 repetitions" in capsys.readouterr().out


# every MLP engine (the engine is chosen per process, hence subprocesses), plus a batch larger than one backward chunk
# (gradients accumulated over several chunks)
VARIANTS = [
    ("tensor-core 3-pass engine", {"STRESS_ENGINE": "tc_3x"}, ["25"]),
    ("tensor-core single-pass engine", {"STRESS_ENGINE": "tc_1x"}, ["25"]),
    ("single-pass weight-gradient engine", {"STRESS_ENGINE": "tc_3x_w1"}, ["25"]),
    ("fp32 SIMT engine", {"STRESS_ENGINE": "simt_fp32"}, ["10"]),
    ("two backward chunks", {}, ["15", "1100", "128"]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("what,env,argv", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_cold_l2_stress_of_selectable_variants(what, env, argv):
    import subprocess
    e = dict(os.environ)
    e.update(env)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "stress_chain.py")] + argv, env=e, capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0 and "stress ok: %s repetitions" % argv[0] in res.stdout, (what, res.stdout[-500:], res.stderr[-1500:])
