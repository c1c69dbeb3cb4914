"""Selects the symbolic-graph backend of the Op layer.

* PyTensor installed → the Ops are genuine PyTensor Ops (drop-in for models written against the
  reference; import list mirrors ``pytensor_federated/op_async.py:4-11`` and
  ``wrapper_ops.py:4-8``).
* PyTensor missing (the offline image) → the in-repo IR :mod:`pytensor_federated_b200.graph`, which
  implements the same names.  Set ``B200FED_GRAPH_BACKEND=builtin`` to force it.
"""
from __future__ import annotations

import os

BACKEND = "builtin"

if os.environ.get("B200FED_GRAPH_BACKEND", "auto") != "builtin":
    try:
        import pytensor
        import pytensor.tensor as at
        from pytensor import function, grad
        from pytensor.compile import optdb
        from pytensor.compile.ops import FromFunctionOp
        from pytensor.gradient import DisconnectedType
        from pytensor.graph import FunctionGraph
        from pytensor.graph.basic import Apply, Variable

        try:
            from pytensor.graph.basic import apply_depends_on
        except ImportError:  # newer PyTensor releases moved the traversal helpers
            try:
                from pytensor.graph.traversal import apply_depends_on
            except ImportError:
                from .graph.core import apply_depends_on  # duck-typed on .inputs / .owner
        from pytensor.graph.features import ReplaceValidate
        from pytensor.graph.op import Op
        from pytensor.graph.rewriting.basic import GraphRewriter

        BACKEND = "pytensor"
    except ModuleNotFoundError:
        pass
    except ImportError as _ex:  # an installed PyTensor whose layout we do not know: say so, use the built-in IR
        import warnings

        warnings.warn(f"PyTensor is installed but could not be used ({_ex}); falling back to the built-in graph IR")
        BACKEND = "builtin"

if BACKEND == "builtin":
    from .graph import core as at  # tensor namespace: scalar, vector, as_tensor, exp, log, sum ...
    from .graph.core import (
        Apply,
        DisconnectedType,
        FromFunctionOp,
        FunctionGraph,
        GraphRewriter,
        Op,
        ReplaceValidate,
        Variable,
        apply_depends_on,
        function,
        grad,
        optdb,
    )

__all__ = [
    "BACKEND", "at", "function", "grad", "optdb", "FromFunctionOp", "DisconnectedType", "FunctionGraph",
    "Apply", "Variable", "apply_depends_on", "ReplaceValidate", "Op", "GraphRewriter",
]
