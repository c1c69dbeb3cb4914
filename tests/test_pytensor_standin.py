"""Drives the PyTensor branch of ``_graph_backend`` against a stand-in package.

PyTensor cannot be installed in this image, so the branch that makes the Ops genuine PyTensor Ops would
otherwise never execute.  The stand-in lays the in-repo IR out under PyTensor's public module paths (the ones
``pytensor_federated/op_async.py:4-11`` and ``wrapper_ops.py:4-8`` import); a fresh interpreter
with the stand-in on its path must select ``BACKEND == "pytensor"``, register ``fuse_asyncs`` in *that* optdb,
and build / differentiate / compile the wrapper Ops through those imports.  It proves the import surface and
the module-level registration, not PyTensor's own semantics."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

STANDIN = {
    "pytensor/__init__.py": "from pytensor_federated_b200.graph.core import function, grad\n__version__ = '0-standin'\n",
    "pytensor/tensor/__init__.py": "from pytensor_federated_b200.graph.core import *  # noqa\n"
                                   "from pytensor_federated_b200.graph.core import as_tensor, constant, scalar, vector, sum, exp, log\n",
    "pytensor/compile/__init__.py": "from pytensor_federated_b200.graph.core import optdb\n",
    "pytensor/compile/ops.py": "from pytensor_federated_b200.graph.core import FromFunctionOp\n",
    "pytensor/gradient.py": "from pytensor_federated_b200.graph.core import DisconnectedType\n",
    "pytensor/graph/__init__.py": "from pytensor_federated_b200.graph.core import FunctionGraph\n",
    "pytensor/graph/basic.py": "from pytensor_federated_b200.graph.core import Apply, Variable, apply_depends_on\n",
    "pytensor/graph/features.py": "from pytensor_federated_b200.graph.core import ReplaceValidate\n",
    "pytensor/graph/op.py": "from pytensor_federated_b200.graph.core import Op\n",
    "pytensor/graph/rewriting/__init__.py": "",
    "pytensor/graph/rewriting/basic.py": "from pytensor_federated_b200.graph.core import GraphRewriter\n",
}

SCRIPT = textwrap.dedent(
    """
    import asyncio, time
    import numpy as np
    import pytensor_federated_b200 as pf               # its graph backend imports `pytensor` (the stand-in) here
    from pytensor_federated_b200 import _graph_backend as gb
    import pytensor, pytensor.tensor as at
    from pytensor.compile import optdb

    assert gb.BACKEND == "pytensor", gb.BACKEND
    assert gb.at is at and gb.optdb is optdb
    assert "fuse_asyncs" in optdb                      # registered at import time, in the backend's optdb

    def logp_grad(a, b):
        x = np.arange(4.0)
        r = x - a - b * x
        return np.asarray(-np.sum(r * r)), [np.asarray(2 * r.sum()), np.asarray(2 * (r * x).sum())]

    a, b = at.scalar("a"), at.scalar("b")
    logp, da, db = pf.LogpGradOp(logp_grad)(a, b)
    ga, gb_ = pytensor.grad(logp, [a, b])
    f = pytensor.function([a, b], [logp, ga, gb_])
    out = f(0.5, 0.25)
    want = logp_grad(0.5, 0.25)
    np.testing.assert_allclose(out[0], want[0]); np.testing.assert_allclose(out[1:], want[1])

    async def slow(x):
        await asyncio.sleep(0.3)
        return np.asarray(x) * 2
    op = pf.op_async.AsyncFromFunctionOp(slow, [at.scalar().type], [at.scalar().type])
    y = op(a) + op(b)
    g = pytensor.function([a, b], [y])              # default mode -> fast_run -> fuse_asyncs
    t0 = time.perf_counter(); (val,) = g(1.0, 2.0); dt = time.perf_counter() - t0
    assert float(val) == 6.0 and dt < 0.55, dt       # the two awaits overlapped
    print("STANDIN-OK")
    """
)


def test_ops_import_and_run_through_the_pytensor_module_layout(tmp_path):
    for rel, body in STANDIN.items():
        path = tmp_path / rel
        path.parent.mkdir(parents=True, exist_ok=True)
        path.write_text(body)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([str(tmp_path), ROOT, env.get("PYTHONPATH", "")])
    env.pop("B200FED_GRAPH_BACKEND", None)
    res = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, env=env, timeout=300)
    assert res.returncode == 0 and "STANDIN-OK" in res.stdout, res.stdout + res.stderr


def test_a_broken_pytensor_install_falls_back_with_a_warning(tmp_path):
    (tmp_path / "pytensor").mkdir()
    (tmp_path / "pytensor" / "__init__.py").write_text("raise ImportError('half-installed')\n")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([str(tmp_path), ROOT, env.get("PYTHONPATH", "")])
    code = ("import warnings\nwith warnings.catch_warnings(record=True) as w:\n    warnings.simplefilter('always')\n"
            "    from pytensor_federated_b200 import _graph_backend as gb\n"
            "assert gb.BACKEND == 'builtin' and any('could not be used' in str(x.message) for x in w)\nprint('FALLBACK-OK')")
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert res.returncode == 0 and "FALLBACK-OK" in res.stdout, res.stdout + res.stderr
