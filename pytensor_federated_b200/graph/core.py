"""A small symbolic graph IR with the slice of PyTensor's API that the federated Ops need.

Why this exists: the reference's L4 layer (``pytensor_federated/op_async.py``,
``wrapper_ops.py``) is written against PyTensor (``Op``, ``Apply``, ``FunctionGraph``,
``optdb``, ``pytensor.grad``, ``DisconnectedType`` — list in SURVEY.md §2.5).  PyTensor is not
available in the offline image, so the same Op sources run on this IR when PyTensor is missing
(see :mod:`pytensor_federated_b200._graph_backend`), which makes ``make_node`` / ``perform`` /
``grad`` / graph fusion executable and testable here, and gives the in-repo samplers
(:mod:`pytensor_federated_b200.sampling`) a differentiable model language.

It is deliberately tiny: dense NumPy evaluation, reverse-mode autodiff over a handful of
elementwise/reduction ops, a merge pass, and an optimiser database with tags and positions.
Names and call signatures follow PyTensor so user code ports in either direction.
"""
from __future__ import annotations

import itertools
import operator
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

# ----------------------------------------------------------------------------- types


class Type:
    def __call__(self, name: Optional[str] = None) -> "Variable":
        return Variable(self, None, None, name)

    def filter(self, value):
        return value


class TensorType(Type):
    def __init__(self, dtype: str = "float64", shape: Tuple[Optional[int], ...] = ()) -> None:
        self.dtype = str(np.dtype(dtype))
        self.shape = tuple(shape)

    @property
    def ndim(self) -> int:
        return len(self.shape)

    def filter(self, value):
        arr = np.asarray(value, dtype=self.dtype)
        if arr.ndim != self.ndim:
            raise TypeError(f"Expected {self.ndim} dimensions, got array of shape {arr.shape}")
        return arr

    def __eq__(self, other) -> bool:
        return isinstance(other, TensorType) and other.dtype == self.dtype and other.ndim == self.ndim

    def __hash__(self) -> int:
        return hash((self.dtype, self.ndim))

    def __repr__(self) -> str:
        return f"TensorType({self.dtype}, shape={self.shape})"


class DisconnectedType(Type):
    """Type of the gradient w.r.t. an output that the cost does not depend on."""

    def __repr__(self) -> str:
        return "DisconnectedType"


class NullType(Type):
    pass


# ----------------------------------------------------------------------------- graph nodes

_var_counter = itertools.count()


class Variable:
    def __init__(self, type: Type, owner: Optional["Apply"], index: Optional[int], name: Optional[str] = None):
        self.type = type
        self.owner = owner
        self.index = index
        self.name = name
        self._id = next(_var_counter)

    # sugar ------------------------------------------------------------------------------
    @property
    def ndim(self) -> int:
        return self.type.ndim

    @property
    def dtype(self) -> str:
        return self.type.dtype

    def __add__(self, other): return add(self, other)
    def __radd__(self, other): return add(other, self)
    def __sub__(self, other): return sub(self, other)
    def __rsub__(self, other): return sub(other, self)
    def __mul__(self, other): return mul(self, other)
    def __rmul__(self, other): return mul(other, self)
    def __truediv__(self, other): return true_div(self, other)
    def __rtruediv__(self, other): return true_div(other, self)
    def __neg__(self): return neg(self)
    def __pow__(self, p): return power(self, p)
    def __getitem__(self, idx): return Subtensor(idx)(self)
    def __iter__(self): raise TypeError("symbolic variables are not iterable")
    def sum(self, axis=None): return Sum(axis)(self)

    def eval(self, inputs_to_values: Optional[Dict["Variable", Any]] = None):
        inputs_to_values = inputs_to_values or {}
        ins = list(inputs_to_values.keys())
        fn = function(ins, self, mode="FAST_COMPILE")
        return fn(*[inputs_to_values[i] for i in ins])

    def __repr__(self) -> str:
        if self.name:
            return self.name
        if self.owner is not None:
            return f"{type(self.owner.op).__name__}.{self.index}"
        return f"<{self.type}>"

    __hash__ = object.__hash__


class Constant(Variable):
    def __init__(self, type: Type, data, name: Optional[str] = None) -> None:
        super().__init__(type, None, None, name)
        self.data = data

    def signature(self):
        arr = np.asarray(self.data)
        return (str(arr.dtype), arr.shape, arr.tobytes())

    def __repr__(self) -> str:
        return self.name or f"Constant({self.data})"


class Apply:
    def __init__(self, op: "Op", inputs: Sequence[Variable], outputs: Sequence[Variable]) -> None:
        self.op = op
        self.inputs = list(inputs)
        self.outputs = list(outputs)
        for i, out in enumerate(self.outputs):
            out.owner = self
            out.index = i

    @property
    def nin(self) -> int:
        return len(self.inputs)

    @property
    def nout(self) -> int:
        return len(self.outputs)

    def __repr__(self) -> str:
        return f"{type(self.op).__name__}({', '.join(map(repr, self.inputs))})"


OutputStorageType = List[List[Optional[Any]]]


class Op:
    """``make_node`` builds the Apply, ``perform`` computes, ``grad`` differentiates."""

    __props__: Tuple[str, ...] = ()
    default_output: Optional[int] = None

    def make_node(self, *inputs) -> Apply:
        raise NotImplementedError

    def perform(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        raise NotImplementedError

    def grad(self, inputs: Sequence[Variable], output_grads: Sequence[Variable]) -> List[Variable]:
        raise NotImplementedError(f"{type(self).__name__} has no grad()")

    def make_thunk(self, node: Apply) -> Optional[Callable]:
        """Optional fast path of a SINGLE-output Op for the compiled :class:`Function`: a callable
        ``f(*input_values) -> output_value`` that does what ``perform`` does without the storage cells.
        ``None`` (the default) makes the Function call ``perform``."""
        return None

    def __call__(self, *inputs, **kwargs):
        node = self.make_node(*inputs)
        if self.default_output is not None:
            return node.outputs[self.default_output]
        if len(node.outputs) == 1:
            return node.outputs[0]
        return list(node.outputs)

    def _props(self):
        return tuple(getattr(self, p) for p in self.__props__)

    def __eq__(self, other) -> bool:
        if self.__props__:
            return type(self) is type(other) and self._props() == other._props()
        return self is other

    def __hash__(self) -> int:
        if self.__props__:
            try:
                return hash((type(self), self._props()))
            except TypeError:
                return hash(type(self))
        return id(self)


# ----------------------------------------------------------------------------- helpers


def as_tensor(x, name: Optional[str] = None, dtype: Optional[str] = None) -> Variable:
    if isinstance(x, Variable):
        return x
    arr = np.asarray(x, dtype=dtype)
    if arr.dtype.kind in "iub" and dtype is None:
        arr = arr.astype("float64") if arr.dtype.kind == "b" else arr
    return Constant(TensorType(arr.dtype, (None,) * arr.ndim), arr, name)


as_tensor_variable = as_tensor


def constant(x, name: Optional[str] = None, dtype: Optional[str] = None) -> Variable:
    """``pytensor.tensor.constant``: a literal in the graph (the reference's gradient-free test pins the
    intercept with ``at.constant(0.5)``)."""
    if isinstance(x, Variable):
        raise TypeError("constant() takes a number or an array, not a graph variable")
    return as_tensor(x, name, dtype)


def scalar(name: Optional[str] = None, dtype: str = "float64") -> Variable:
    return TensorType(dtype, ())(name)


def vector(name: Optional[str] = None, dtype: str = "float64") -> Variable:
    return TensorType(dtype, (None,))(name)


def matrix(name: Optional[str] = None, dtype: str = "float64") -> Variable:
    return TensorType(dtype, (None, None))(name)


dscalar, dvector, dmatrix = scalar, vector, matrix


def _out_type(*inputs: Variable) -> TensorType:
    nd = max(i.type.ndim for i in inputs)
    dt = np.result_type(*[i.type.dtype for i in inputs])
    return TensorType(dt, (None,) * nd)


_SCALAR_OPERATORS = {"add": operator.add, "sub": operator.sub, "mul": operator.mul, "true_div": operator.truediv,
                     "neg": operator.neg}


_SCALAR_INFIX = {"add": "({0} + {1})", "sub": "({0} - {1})", "mul": "({0} * {1})", "true_div": "({0} / {1})", "neg": "(-{0})"}


class Elemwise(Op):
    """Broadcasting NumPy ufunc with a hand-written derivative."""

    __props__ = ("name",)

    def __init__(self, name: str, fn: Callable, grad_fn: Callable, float_out: bool = False) -> None:
        self.name = name
        self._fn = fn
        self._grad_fn = grad_fn
        self._float_out = float_out

    def make_node(self, *inputs) -> Apply:
        ins = [as_tensor(i) for i in inputs]
        t = _out_type(*ins)
        if self._float_out and np.dtype(t.dtype).kind in "iub":
            t = TensorType("float64", t.shape)
        return Apply(self, ins, [t()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.asarray(self._fn(*inputs), dtype=node.outputs[0].type.dtype)

    def make_thunk(self, node):
        fn, dt, asarray = self._fn, np.dtype(node.outputs[0].type.dtype), np.asarray
        if dt.kind == "f" and node.outputs[0].type.ndim == 0 and \
                all(isinstance(i.type, TensorType) and i.type.ndim == 0 for i in node.inputs):
            # statically scalar: NumPy scalars instead of 0-d arrays (scalar arithmetic is several times cheaper
            # than a ufunc call on 0-d arrays); the Function hands 0-d arrays to every other kind of consumer
            sc = dt.type
            f = _SCALAR_OPERATORS.get(self.name, fn)

            def scalar_thunk(*inputs):
                out = f(*inputs)
                return out if type(out) is sc else sc(out)

            scalar_thunk.returns_scalar = True
            # float64 (op) float64 is float64: the generated code can write the operator out instead of calling
            if self.name in _SCALAR_INFIX and dt == np.float64 and all(i.type.dtype == "float64" for i in node.inputs):
                scalar_thunk.inline = _SCALAR_INFIX[self.name]
            return scalar_thunk

        def thunk(*inputs):
            out = fn(*inputs)
            # the ufunc of arrays of the declared dtype already returns the right thing; anything else is converted
            return out if type(out) is np.ndarray and out.dtype == dt else asarray(out, dtype=dt)

        return thunk

    def grad(self, inputs, output_grads):
        (g,) = output_grads
        out = self(*inputs)
        return [reduce_to(gi, x) for gi, x in zip(self._grad_fn(inputs, out, g), inputs)]


class ReduceTo(Op):
    """Sums ``g`` down to the runtime shape of ``like`` (undoes broadcasting in backprop)."""

    __props__ = ()

    def make_node(self, g, like) -> Apply:
        g, like = as_tensor(g), as_tensor(like)
        return Apply(self, [g, like], [TensorType(g.type.dtype, like.type.shape)()])

    def perform(self, node, inputs, output_storage) -> None:
        g, like = inputs
        g = np.asarray(g)
        shape = np.shape(like)
        while g.ndim > len(shape):
            g = g.sum(axis=0)
        for ax, n in enumerate(shape):
            if n == 1 and g.shape[ax] != 1:
                g = g.sum(axis=ax, keepdims=True)
        output_storage[0][0] = np.asarray(g, dtype=node.outputs[0].type.dtype).reshape(shape)

    def make_thunk(self, node):
        dt, asarray, np_shape, perform = np.dtype(node.outputs[0].type.dtype), np.asarray, np.shape, self.perform

        def thunk(g, like):
            if np_shape(g) == np_shape(like):          # nothing was broadcast: the usual case at run time
                return g if type(g) is np.ndarray and g.dtype == dt else asarray(g, dtype=dt)
            cell = [[None]]
            perform(node, [g, like], cell)
            return cell[0][0]

        return thunk

    def grad(self, inputs, output_grads):
        g, like = inputs
        (gz,) = output_grads
        return [gz + zeros_like(g), DisconnectedType()()]


def reduce_to(g: Variable, like: Variable) -> Variable:
    if isinstance(g.type, DisconnectedType):
        return g
    if g.type.ndim == like.type.ndim == 0:
        return g
    return ReduceTo()(g, like)


class Sum(Op):
    __props__ = ("axis",)

    def __init__(self, axis=None) -> None:
        self.axis = axis

    def make_node(self, x) -> Apply:
        x = as_tensor(x)
        nd = 0 if self.axis is None else x.type.ndim - 1
        return Apply(self, [x], [TensorType(x.type.dtype, (None,) * nd)()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.asarray(np.sum(inputs[0], axis=self.axis))

    def make_thunk(self, node):
        axis, np_sum, asarray, ndarray = self.axis, np.sum, np.asarray, np.ndarray
        # the method skips np.sum's dispatch wrappers (a third of the cost on the short vectors of a model graph)
        return lambda x: asarray(x.sum(axis=axis) if type(x) is ndarray else np_sum(x, axis=axis))

    def grad(self, inputs, output_grads):
        (x,) = inputs
        (g,) = output_grads
        if self.axis is None:
            return [g + zeros_like(x)]
        return [ExpandDims(self.axis)(g) + zeros_like(x)]


class ExpandDims(Op):
    __props__ = ("axis",)

    def __init__(self, axis: int) -> None:
        self.axis = axis

    def make_node(self, x) -> Apply:
        x = as_tensor(x)
        return Apply(self, [x], [TensorType(x.type.dtype, (None,) * (x.type.ndim + 1))()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.expand_dims(inputs[0], self.axis)

    def grad(self, inputs, output_grads):
        return [Sum(self.axis)(output_grads[0])]


class Subtensor(Op):
    """``x[idx]`` with a static integer or slice index."""

    __props__ = ("idx_key",)

    def __init__(self, idx) -> None:
        self.idx = idx
        self.idx_key = repr(idx)

    def make_node(self, x) -> Apply:
        x = as_tensor(x)
        idx = self.idx if isinstance(self.idx, tuple) else (self.idx,)
        # NB: ``sum`` is shadowed by the symbolic sum of this module
        dropped = len([i for i in idx if isinstance(i, (int, np.integer))])
        added = len([i for i in idx if i is None])
        return Apply(self, [x], [TensorType(x.type.dtype, (None,) * (x.type.ndim - dropped + added))()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.asarray(inputs[0][self.idx])

    def make_thunk(self, node):
        idx, asarray = self.idx, np.asarray
        return lambda x: asarray(x[idx])

    def grad(self, inputs, output_grads):
        return [IncSubtensorZeros(self.idx)(inputs[0], output_grads[0])]


class IncSubtensorZeros(Op):
    __props__ = ("idx_key",)

    def __init__(self, idx) -> None:
        self.idx = idx
        self.idx_key = repr(idx)

    def make_node(self, like, g) -> Apply:
        like, g = as_tensor(like), as_tensor(g)
        return Apply(self, [like, g], [like.type()])

    def perform(self, node, inputs, output_storage) -> None:
        like, g = inputs
        out = np.zeros(np.shape(like), dtype=node.outputs[0].type.dtype)
        out[self.idx] = g
        output_storage[0][0] = out

    def make_thunk(self, node):
        idx, dt, zeros, np_shape = self.idx, np.dtype(node.outputs[0].type.dtype), np.zeros, np.shape

        def thunk(like, g):
            out = zeros(np_shape(like), dtype=dt)
            out[idx] = g
            return out

        return thunk

    def grad(self, inputs, output_grads):
        return [DisconnectedType()(), Subtensor(self.idx)(output_grads[0])]


class ScatterAdd(Op):
    """``zeros_like(like)`` with ``out[idx_k] += g_k`` for every ``(idx_k, g_k)`` — what a sum of
    :class:`IncSubtensorZeros` terms computes, in one allocation (built by :class:`IncSubtensorMerger`: the
    gradient w.r.t. a vector whose elements are used one by one, e.g. one intercept per federated node)."""

    __props__ = ("idx_keys",)

    def __init__(self, idxs) -> None:
        self.idxs = tuple(idxs)
        self.idx_keys = tuple(repr(i) for i in self.idxs)

    def make_node(self, like, *gs) -> Apply:
        if len(gs) != len(self.idxs):
            raise ValueError(f"ScatterAdd expects {len(self.idxs)} increments, got {len(gs)}")
        like = as_tensor(like)
        return Apply(self, [like, *[as_tensor(g) for g in gs]], [like.type()])

    def perform(self, node, inputs, output_storage) -> None:
        like, *gs = inputs
        out = np.zeros(np.shape(like), dtype=node.outputs[0].type.dtype)
        for idx, g in zip(self.idxs, gs):
            out[idx] += g
        output_storage[0][0] = out

    def make_thunk(self, node):
        idxs, dt, zeros, np_shape = self.idxs, np.dtype(node.outputs[0].type.dtype), np.zeros, np.shape

        def thunk(like, *gs):
            out = zeros(np_shape(like), dtype=dt)
            for idx, g in zip(idxs, gs):
                out[idx] += g
            return out

        return thunk

    def grad(self, inputs, output_grads):
        (gz,) = output_grads
        return [DisconnectedType()(), *[Subtensor(idx)(gz) for idx in self.idxs]]


class ZerosLike(Op):
    __props__ = ()

    def make_node(self, x) -> Apply:
        x = as_tensor(x)
        dt = x.type.dtype if np.dtype(x.type.dtype).kind == "f" else "float64"
        return Apply(self, [x], [TensorType(dt, x.type.shape)()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.zeros(np.shape(inputs[0]), dtype=node.outputs[0].type.dtype)

    def make_thunk(self, node):
        dt, zeros, np_shape = np.dtype(node.outputs[0].type.dtype), np.zeros, np.shape
        return lambda x: zeros(np_shape(x), dtype=dt)

    def grad(self, inputs, output_grads):
        return [DisconnectedType()()]


def zeros_like(x) -> Variable:
    return ZerosLike()(x)


class Stack(Op):
    """Stacks equally shaped tensors (typically scalars) along a new leading axis (``at.stack``)."""

    __props__ = ()

    def make_node(self, *xs) -> Apply:
        xs = [as_tensor(x) for x in xs]
        nd = max(x.type.ndim for x in xs)
        return Apply(self, xs, [TensorType("float64", (None,) * (nd + 1))()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.stack([np.asarray(x, dtype=np.float64) for x in inputs], axis=0)

    def grad(self, inputs, output_grads):
        (g,) = output_grads
        return [g[i] for i in range(len(inputs))]


def stack(xs) -> Variable:
    return Stack()(*xs)


_add = Elemwise("add", np.add, lambda ins, out, g: [g, g])
_sub = Elemwise("sub", np.subtract, lambda ins, out, g: [g, neg(g)])
_mul = Elemwise("mul", np.multiply, lambda ins, out, g: [g * ins[1], g * ins[0]])
_div = Elemwise("true_div", np.true_divide, lambda ins, out, g: [g / ins[1], neg(g * ins[0] / (ins[1] * ins[1]))], True)
_neg = Elemwise("neg", np.negative, lambda ins, out, g: [neg(g)])
_exp = Elemwise("exp", np.exp, lambda ins, out, g: [g * out], True)
_log = Elemwise("log", np.log, lambda ins, out, g: [g / ins[0]], True)
_sqr = Elemwise("sqr", np.square, lambda ins, out, g: [g * 2.0 * ins[0]])
_sqrt = Elemwise("sqrt", np.sqrt, lambda ins, out, g: [g / (2.0 * out)], True)
_sigmoid = Elemwise("sigmoid", lambda x: 1.0 / (1.0 + np.exp(-x)), lambda ins, out, g: [g * out * (1.0 - out)], True)
_softplus = Elemwise("softplus", lambda x: np.logaddexp(0.0, x), lambda ins, out, g: [g * sigmoid(ins[0])], True)


_tanh = Elemwise("tanh", np.tanh, lambda ins, out, g: [g * (1.0 - out * out)], True)
_log1p = Elemwise("log1p", np.log1p, lambda ins, out, g: [g / (1.0 + ins[0])], True)
_abs = Elemwise("abs", np.abs, lambda ins, out, g: [g * _sign(ins[0])])
_sign = Elemwise("sign", np.sign, lambda ins, out, g: [zeros_like(ins[0])])
_maximum = Elemwise("maximum", np.maximum,
                    lambda ins, out, g: [g * _ge(ins[0], ins[1]), g * (1.0 - _ge(ins[0], ins[1]))])
_ge = Elemwise("ge", lambda a, b: (np.asarray(a) >= np.asarray(b)).astype(np.float64),
               lambda ins, out, g: [zeros_like(ins[0]), zeros_like(ins[1])], True)


class Dot(Op):
    """``dot(a, b)`` for vectors and matrices (NumPy semantics for 1-d / 2-d operands)."""

    __props__ = ()

    def make_node(self, a, b) -> Apply:
        a, b = as_tensor(a), as_tensor(b)
        if not (1 <= a.type.ndim <= 2 and 1 <= b.type.ndim <= 2):
            raise TypeError("dot supports vectors and matrices")
        nd = a.type.ndim + b.type.ndim - 2
        return Apply(self, [a, b], [TensorType(np.result_type(a.type.dtype, b.type.dtype), (None,) * nd)()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.asarray(np.dot(*inputs), dtype=node.outputs[0].type.dtype)

    def grad(self, inputs, output_grads):
        a, b = inputs
        (g,) = output_grads
        na, nb = a.type.ndim, b.type.ndim
        if na == 1 and nb == 1:
            return [g * b, g * a]
        if na == 2 and nb == 1:          # (m,k).(k,) -> (m,)
            return [ExpandDims(1)(g) * ExpandDims(0)(b), Dot()(Transpose()(a), g)]
        if na == 1 and nb == 2:          # (k,).(k,n) -> (n,)
            return [Dot()(b, g), ExpandDims(1)(a) * ExpandDims(0)(g)]
        return [Dot()(g, Transpose()(b)), Dot()(Transpose()(a), g)]


class Transpose(Op):
    __props__ = ()

    def make_node(self, x) -> Apply:
        x = as_tensor(x)
        return Apply(self, [x], [x.type()])

    def perform(self, node, inputs, output_storage) -> None:
        output_storage[0][0] = np.ascontiguousarray(np.transpose(inputs[0]))

    def grad(self, inputs, output_grads):
        return [Transpose()(output_grads[0])]


def dot(a, b): return Dot()(a, b)
def transpose(x): return Transpose()(x)
def tanh(a): return _tanh(a)
def log1p(a): return _log1p(a)
def abs(a): return _abs(a)  # noqa: A001 - mirrors pytensor.tensor.abs
def maximum(a, b): return _maximum(a, b)


def mean(x, axis=None):
    x = as_tensor(x)
    total = x.sum(axis)
    return total / _size_like(x, axis)


class _SizeAlong(Op):
    """Number of elements reduced by ``sum(axis)`` as a float scalar (runtime shape)."""

    __props__ = ("axis",)

    def __init__(self, axis=None) -> None:
        self.axis = axis

    def make_node(self, x) -> Apply:
        return Apply(self, [as_tensor(x)], [TensorType("float64", ())()])

    def perform(self, node, inputs, output_storage) -> None:
        shape = np.shape(inputs[0])
        output_storage[0][0] = np.asarray(float(np.prod(shape) if self.axis is None else shape[self.axis]))

    def grad(self, inputs, output_grads):
        return [zeros_like(inputs[0])]


def _size_like(x, axis):
    return _SizeAlong(axis)(x)


def add(a, b): return _add(a, b)
def sub(a, b): return _sub(a, b)
def mul(a, b): return _mul(a, b)
def true_div(a, b): return _div(a, b)
def neg(a): return _neg(a)
def exp(a): return _exp(a)
def log(a): return _log(a)
def sqr(a): return _sqr(a)
def sqrt(a): return _sqrt(a)
def sigmoid(a): return _sigmoid(a)
def softplus(a): return _softplus(a)


def power(a, p):
    if isinstance(p, (int, float)) and p == 2:
        return sqr(a)
    return exp(as_tensor(float(p)) * log(a)) if isinstance(p, (int, float)) else exp(p * log(a))


def sum(x, axis=None):  # noqa: A001 - mirrors pytensor.tensor.sum
    return as_tensor(x).sum(axis)


# ----------------------------------------------------------------------------- traversal


def ancestors_applies(outputs: Iterable[Variable]) -> List[Apply]:
    """Apply nodes needed for ``outputs`` in a deterministic topological order."""
    order: List[Apply] = []
    seen = set()
    stack_: List[Tuple[Apply, int]] = []
    for out in outputs:
        if out.owner is not None and id(out.owner) not in seen:
            stack_.append((out.owner, 0))
            while stack_:
                node, i = stack_.pop()
                if id(node) in seen:
                    continue
                if i < len(node.inputs):
                    stack_.append((node, i + 1))
                    parent = node.inputs[i].owner
                    if parent is not None and id(parent) not in seen:
                        stack_.append((parent, 0))
                else:
                    seen.add(id(node))
                    order.append(node)
    return order


def apply_depends_on(apply: Apply, depends_on: Union[Apply, Sequence[Apply]]) -> bool:
    """True when ``apply`` (transitively) consumes an output of ``depends_on``."""
    targets = {id(depends_on)} if hasattr(depends_on, "inputs") else {id(d) for d in depends_on}
    seen = set()
    todo = [apply]
    while todo:
        node = todo.pop()
        for inp in node.inputs:
            parent = inp.owner
            if parent is None or id(parent) in seen:
                continue
            if id(parent) in targets:
                return True
            seen.add(id(parent))
            todo.append(parent)
    return False


# ----------------------------------------------------------------------------- autodiff


def grad(cost: Variable, wrt: Union[Variable, Sequence[Variable]], disconnected_inputs: str = "zero"):
    """Reverse-mode gradient of a scalar ``cost``.

    Outputs the cost does not depend on receive a ``DisconnectedType`` gradient variable, which
    is how ``LogpGradOp.grad`` recognises that nobody differentiates through its gradient
    outputs (reference: ``wrapper_ops.py:122-125``).
    """
    single = isinstance(wrt, Variable)
    wrts = [wrt] if single else list(wrt)
    if cost.type.ndim != 0:
        raise TypeError("grad() needs a scalar cost")
    grads: Dict[int, Variable] = {id(cost): as_tensor(1.0)}
    keep = {id(cost): cost}
    for node in reversed(ancestors_applies([cost])):
        if not any(id(o) in grads for o in node.outputs):
            continue
        ogs = [grads.get(id(o)) if id(o) in grads else DisconnectedType()() for o in node.outputs]
        igs = node.op.grad(node.inputs, ogs)
        if len(igs) != len(node.inputs):
            raise ValueError(f"{type(node.op).__name__}.grad returned {len(igs)} gradients for {len(node.inputs)} inputs")
        for inp, g in zip(node.inputs, igs):
            if g is None or isinstance(g.type, (DisconnectedType, NullType)):
                continue
            if id(inp) in grads:
                grads[id(inp)] = grads[id(inp)] + g
            else:
                grads[id(inp)] = g
                keep[id(inp)] = inp
    result = []
    for w in wrts:
        if id(w) in grads:
            result.append(grads[id(w)])
        elif disconnected_inputs == "raise":
            raise ValueError(f"{w} is not part of the cost's graph")
        else:
            result.append(zeros_like(w))
    return result[0] if single else result


# ----------------------------------------------------------------------------- FunctionGraph


class Feature:
    def on_attach(self, fgraph: "FunctionGraph") -> None:
        pass


class ReplaceValidate(Feature):
    """Adds ``replace_all_validate``: apply replacements, roll back if the graph breaks."""

    def on_attach(self, fgraph: "FunctionGraph") -> None:
        if hasattr(fgraph, "replace_all_validate"):
            return

        def replace_all_validate(pairs, reason=None):
            snapshot = fgraph._snapshot()
            try:
                fgraph.replace_all(pairs, reason=reason)
                fgraph.toposort()  # raises on cycles / dangling inputs
            except Exception:
                fgraph._restore(snapshot)
                raise

        fgraph.replace_all_validate = replace_all_validate


class FunctionGraph:
    def __init__(self, inputs: Sequence[Variable], outputs: Sequence[Variable], clone: bool = True) -> None:
        if clone:
            inputs, outputs = clone_graph(inputs, outputs)
        self.inputs = list(inputs)
        self.outputs = list(outputs)
        self._features: List[Feature] = []

    def attach_feature(self, feature: Feature) -> None:
        if any(type(f) is type(feature) for f in self._features):
            return
        self._features.append(feature)
        feature.on_attach(self)

    @property
    def apply_nodes(self) -> List[Apply]:
        return ancestors_applies(self.outputs)

    def toposort(self) -> List[Apply]:
        order = ancestors_applies(self.outputs)
        known = {id(v) for v in self.inputs}
        for node in order:
            for inp in node.inputs:
                if inp.owner is None and not isinstance(inp, Constant) and id(inp) not in known:
                    raise ValueError(f"Graph input {inp} is not an input of the FunctionGraph")
        return order

    def replace_all(self, pairs, reason=None) -> None:
        mapping = {id(old): new for old, new in pairs}
        if not mapping:
            return
        for node in ancestors_applies(self.outputs):
            for i, inp in enumerate(node.inputs):
                if id(inp) in mapping:
                    node.inputs[i] = mapping[id(inp)]
        for i, out in enumerate(self.outputs):
            if id(out) in mapping:
                self.outputs[i] = mapping[id(out)]
        # replacements may themselves consume replaced variables (none of ours do); re-run once
        for node in ancestors_applies(self.outputs):
            for i, inp in enumerate(node.inputs):
                if id(inp) in mapping and mapping[id(inp)] is not inp:
                    node.inputs[i] = mapping[id(inp)]

    def replace(self, old: Variable, new: Variable, reason=None) -> None:
        self.replace_all([(old, new)], reason=reason)

    def _snapshot(self):
        return list(self.outputs), [(n, list(n.inputs)) for n in ancestors_applies(self.outputs)]

    def _restore(self, snap) -> None:
        outputs, nodes = snap
        self.outputs = outputs
        for node, inputs in nodes:
            node.inputs = inputs


def clone_graph(inputs: Sequence[Variable], outputs: Sequence[Variable]):
    """Copies the Apply nodes between ``inputs`` and ``outputs`` (Ops are shared)."""
    memo: Dict[int, Variable] = {}
    new_inputs = []
    for v in inputs:
        nv = Variable(v.type, None, None, v.name)
        memo[id(v)] = nv
        new_inputs.append(nv)
    for node in ancestors_applies(outputs):
        ins = []
        for inp in node.inputs:
            if id(inp) not in memo:
                memo[id(inp)] = inp  # constants and free variables are shared
            ins.append(memo[id(inp)])
        outs = [Variable(o.type, None, None, o.name) for o in node.outputs]
        Apply(node.op, ins, outs)
        for o, no in zip(node.outputs, outs):
            memo[id(o)] = no
    return new_inputs, [memo.get(id(o), o) for o in outputs]


# ----------------------------------------------------------------------------- rewriting


class GraphRewriter:
    def add_requirements(self, fgraph: FunctionGraph) -> None:
        pass

    def apply(self, fgraph: FunctionGraph) -> None:
        raise NotImplementedError

    def rewrite(self, fgraph: FunctionGraph) -> None:
        self.add_requirements(fgraph)
        self.apply(fgraph)


class MergeOptimizer(GraphRewriter):
    """Deduplicates equal constants and Apply nodes with equal op and identical inputs.

    This is what makes ``LogpGradOp.grad`` cost no second remote call: its re-application of
    the same Op instance to the same inputs is merged into the forward node.
    """

    def apply(self, fgraph: FunctionGraph) -> None:
        changed = True
        while changed:
            changed = False
            const_seen: Dict[Any, Variable] = {}
            node_seen: Dict[Any, Apply] = {}
            pairs = []
            for node in fgraph.toposort():
                for i, inp in enumerate(node.inputs):
                    if isinstance(inp, Constant):
                        sig = inp.signature()
                        if sig in const_seen and const_seen[sig] is not inp:
                            node.inputs[i] = const_seen[sig]
                        else:
                            const_seen.setdefault(sig, inp)
                try:
                    key = (node.op, tuple(id(i) for i in node.inputs))
                    hash(key)
                except TypeError:
                    continue
                other = node_seen.get(key)
                if other is None:
                    node_seen[key] = node
                elif other is not node:
                    pairs.extend(zip(node.outputs, other.outputs))
            if pairs:
                fgraph.replace_all(pairs, reason="merge")
                changed = True


class IdentityEliminator(GraphRewriter):
    """Removes the arithmetic no-ops that reverse-mode differentiation leaves behind — ``g + zeros_like(x)`` for a
    scalar ``x``, ``1.0 * g``, ``g + 0.0`` — whenever the surviving operand already has the node's type (dtype
    and rank), so values, dtypes and shapes are untouched.  The gradient graph of a model with a few dozen
    scalar terms loses about half of its nodes, which a sampler pays for at every model evaluation."""

    @staticmethod
    def _is_scalar_const(v: Variable, value: float) -> bool:
        return isinstance(v, Constant) and np.ndim(v.data) == 0 and np.asarray(v.data).dtype.kind in "fiu" \
            and float(v.data) == value

    @staticmethod
    def _is_scalar_zeros(v: Variable) -> bool:
        node = v.owner
        return node is not None and isinstance(node.op, ZerosLike) and node.inputs[0].type.ndim == 0

    def apply(self, fgraph: FunctionGraph) -> None:
        changed = True
        while changed:
            changed = False
            pairs = []
            for node in fgraph.toposort():
                op = node.op
                if not isinstance(op, Elemwise) or len(node.inputs) != 2 or op.name not in ("add", "mul"):
                    continue
                out = node.outputs[0]
                for keep, other in ((node.inputs[0], node.inputs[1]), (node.inputs[1], node.inputs[0])):
                    if not isinstance(keep.type, TensorType) or keep.type.dtype != out.type.dtype \
                            or keep.type.ndim != out.type.ndim:
                        continue
                    neutral = (self._is_scalar_const(other, 0.0) or self._is_scalar_zeros(other)) if op.name == "add" \
                        else self._is_scalar_const(other, 1.0)
                    if neutral:
                        pairs.append((out, keep))
                        break
            if pairs:
                # one replacement may feed another (a + 0 + 0): resolve chains before rewiring
                target = {id(old): new for old, new in pairs}
                resolved = []
                for old, new in pairs:
                    while id(new) in target:
                        new = target[id(new)]
                    resolved.append((old, new))
                fgraph.replace_all(resolved, reason="identity")
                changed = True


class IncSubtensorMerger(GraphRewriter):
    """``inc(like, g0)[i0] + inc(like, g1)[i1] + ... (+ other terms)`` -> ``ScatterAdd(like, g0, g1, ...) (+ other
    terms)``: the gradient of ``sum_k f_k(x[i_k])`` w.r.t. ``x`` costs one allocation instead of one vector of zeros
    and one vector addition per term."""

    @staticmethod
    def _is_add(node) -> bool:
        return node is not None and isinstance(node.op, Elemwise) and node.op.name == "add" and len(node.inputs) == 2

    def apply(self, fgraph: FunctionGraph) -> None:
        order = fgraph.toposort()
        clients: Dict[int, List[Apply]] = {}
        for node in order:
            for inp in node.inputs:
                clients.setdefault(id(inp), []).append(node)
        outputs = {id(o) for o in fgraph.outputs}
        pairs = []
        for node in order:
            if not self._is_add(node):
                continue
            out = node.outputs[0]
            if any(self._is_add(c) for c in clients.get(id(out), [])) and id(out) not in outputs:
                continue                                  # an inner node of a larger sum: handled from its top
            leaves: List[Variable] = []

            def collect(v: Variable, top: bool) -> None:
                n = v.owner
                # descend only through sums nobody else needs (and that are not outputs themselves)
                if self._is_add(n) and (top or (len(clients.get(id(v), [])) == 1 and id(v) not in outputs)) \
                        and n.inputs[0].type == v.type and n.inputs[1].type == v.type:
                    collect(n.inputs[0], False)
                    collect(n.inputs[1], False)
                else:
                    leaves.append(v)

            collect(out, True)
            groups: Dict[int, List[Variable]] = {}
            for leaf in leaves:
                n = leaf.owner
                if n is not None and isinstance(n.op, IncSubtensorZeros) and leaf.type == out.type:
                    groups.setdefault(id(n.inputs[0]), []).append(leaf)
            groups = {k: v for k, v in groups.items() if len(v) >= 2}
            if not groups:
                continue
            merged_ids = {id(leaf) for group in groups.values() for leaf in group}
            terms: List[Variable] = [leaf for leaf in leaves if id(leaf) not in merged_ids]
            for group in groups.values():
                like = group[0].owner.inputs[0]
                scatter = ScatterAdd([leaf.owner.op.idx for leaf in group])(like, *[leaf.owner.inputs[1] for leaf in group])
                if scatter.type != out.type:
                    terms = None
                    break
                terms.append(scatter)
            if not terms:
                continue
            total = terms[0]
            for t in terms[1:]:
                total = total + t
            if total.type == out.type:
                pairs.append((out, total))
        if pairs:
            fgraph.replace_all(pairs, reason="merge-inc-subtensor")


class OptimizerDB:
    """Named rewriters with tags and positions (``pytensor.compile.optdb`` subset)."""

    def __init__(self) -> None:
        self._entries: Dict[str, Tuple[GraphRewriter, Tuple[str, ...], float]] = {}

    def register(self, name: str, rewriter: GraphRewriter, *tags: str, position: float = 50.0) -> None:
        if name in self._entries:
            raise ValueError(f"The name {name!r} is already registered.")
        self._entries[name] = (rewriter, tuple(tags), float(position))

    def __contains__(self, name: str) -> bool:
        return name in self._entries

    def __getitem__(self, name: str) -> GraphRewriter:
        return self._entries[name][0]

    def remove(self, name: str) -> None:
        self._entries.pop(name, None)

    def query(self, *tags: str, exclude: Sequence[str] = ()) -> List[GraphRewriter]:
        picked = [
            (pos, name, rw)
            for name, (rw, t, pos) in self._entries.items()
            if name not in exclude and any(tag in t for tag in tags)
        ]
        return [rw for _, _, rw in sorted(picked, key=lambda e: (e[0], e[1]))]


optdb = OptimizerDB()
optdb.register("merge1", MergeOptimizer(), "fast_run", "fast_compile", position=0)
optdb.register("identities", IdentityEliminator(), "fast_run", position=10)
optdb.register("merge_inc_subtensor", IncSubtensorMerger(), "fast_run", position=20)
optdb.register("merge2", MergeOptimizer(), "fast_run", position=49)

MODES = {"FAST_RUN": "fast_run", "FAST_COMPILE": "fast_compile"}
default_mode = "FAST_RUN"


class Mode:
    def __init__(self, name: str = "FAST_RUN", excluding: Sequence[str] = ()) -> None:
        self.name = name
        self._excluding = tuple(excluding)

    def excluding(self, *names: str) -> "Mode":
        return Mode(self.name, self._excluding + names)


def get_mode(mode) -> Mode:
    if isinstance(mode, Mode):
        return mode
    return Mode(mode or default_mode)


# ----------------------------------------------------------------------------- compilation


class Function:
    """The compiled graph: every variable gets a slot (constants are pre-filled), every Apply node becomes one
    step — a thunk (``Op.make_thunk``) where the Op offers one, else ``perform`` with fresh storage cells — and
    the steps are emitted as ONE generated straight-line Python function.  Statically scalar float arithmetic
    runs on NumPy scalars (``scalar_thunk``: several times cheaper than ufunc calls on 0-d arrays); a value is
    converted once (``x[()]`` / ``asarray``) where a consumer of the other kind needs it.  This is the per-model-
    evaluation overhead a sampler pays on top of the federated launch."""

    _ARRAY, _SCALAR = 0, 1

    def __init__(self, fgraph: FunctionGraph, single_output: bool) -> None:
        self.fgraph = fgraph
        self.maker = self  # pytensor spelling: fn.maker.fgraph
        self._single = single_output
        self._order = fgraph.toposort()
        slots: Dict[int, int] = {}
        template: List[Any] = []

        def slot_of(v: Variable) -> int:
            k = slots.get(id(v))
            if k is None:
                k = slots[id(v)] = len(template)
                template.append(v.data if isinstance(v, Constant) else None)
            return k

        self._in_slots = [slot_of(v) for v in fgraph.inputs]
        self._filters = [v.type.filter for v in fgraph.inputs]
        form: Dict[int, int] = {}          # slot -> form its producer leaves it in (default: array)
        steps = []
        for node in self._order:
            ins = tuple(slot_of(i) for i in node.inputs)
            outs = tuple(slot_of(o) for o in node.outputs)
            thunk = node.op.make_thunk(node) if len(outs) == 1 else None
            wants = self._SCALAR if getattr(thunk, "returns_scalar", False) else self._ARRAY
            # per input: None = as it is, else the form to convert to
            conv = tuple(None if form.get(i, self._ARRAY) == wants else wants for i in ins)
            if thunk is not None:
                steps.append((thunk, None, ins, outs[0], conv))
                form[outs[0]] = wants
            else:
                steps.append((node.op.perform, node, ins, outs, conv))
        self._steps = steps
        self._out_slots = [slot_of(o) for o in fgraph.outputs]
        self._out_conv = [self._ARRAY if form.get(k, self._ARRAY) == self._SCALAR else None for k in self._out_slots]
        self._template = template
        self._keep = [v for node in self._order for v in node.inputs]   # ids stay unique while the plan lives
        self._run = self._generate()

    def _generate(self) -> Optional[Callable]:
        """``def _run(v0, v1): v7 = f3(v1, c4); ...; return [v30, v31]`` with constants, thunks and ``perform``
        methods bound as globals (``__call__`` falls back to an interpreter loop if this is not possible)."""
        ns: Dict[str, Any] = {"_A": np.asarray}
        const_slots = {k for k, v in enumerate(self._template) if v is not None}
        converted: Dict[Tuple[int, int], str] = {}   # (slot, form) -> name of the converted value
        for k in const_slots:
            ns[f"c{k}"] = self._template[k]
        base = lambda k: f"c{k}" if k in const_slots else f"v{k}"
        args = [f"v{k}" for k in self._in_slots]
        if len(set(args)) != len(args):
            return None
        lines = [f"def _run({', '.join(args)}):"]

        def operand(k: int, to) -> str:
            if to is None:
                return base(k)
            name = converted.get((k, to))
            if name is None:
                name = converted[(k, to)] = f"{base(k)}{'s' if to == self._SCALAR else 'a'}"
                expr = f"{base(k)}[()]" if to == self._SCALAR else f"_A({base(k)})"
                if k in const_slots:
                    ns[name] = eval(expr, ns)  # noqa: S307 - a constant of the plan, converted once
                else:
                    lines.append(f"    {name} = {expr}")
            return name

        for n, (fn, node, ins, outs, conv) in enumerate(self._steps):
            ns[f"f{n}"] = fn
            operands = [operand(i, c) for i, c in zip(ins, conv)]
            call_args = ", ".join(operands)
            inline = getattr(fn, "inline", None) if node is None else None
            if inline is not None:
                lines.append(f"    v{outs} = {inline.format(*operands)}")
            elif node is None:
                lines.append(f"    v{outs} = f{n}({call_args})")
            else:
                ns[f"n{n}"] = node
                lines.append(f"    s = [{', '.join('[None]' for _ in outs)}]")
                lines.append(f"    f{n}(n{n}, [{call_args}], s)")
                for j, k in enumerate(outs):
                    lines.append(f"    v{k} = s[{j}][0]")
        lines.append(f"    return [{', '.join([operand(k, c) for k, c in zip(self._out_slots, self._out_conv)])}]")
        try:
            exec(compile("\n".join(lines), "<pytensor_federated_b200.graph.Function>", "exec"), ns)  # noqa: S102 - own plan
        except (SyntaxError, MemoryError, RecursionError):
            return None
        return ns["_run"]

    def _convert(self, value, to):
        if to is None:
            return value
        return np.asarray(value)[()] if to == self._SCALAR else np.asarray(value)

    def __call__(self, *args):
        if len(args) != len(self._in_slots):
            raise TypeError(f"Expected {len(self._in_slots)} inputs, got {len(args)}")
        if self._run is not None:
            results = self._run(*[flt(arg) for flt, arg in zip(self._filters, args)])
            return results[0] if self._single else results
        vals = list(self._template)
        for k, flt, arg in zip(self._in_slots, self._filters, args):
            vals[k] = flt(arg)
        for fn, node, ins, outs, conv in self._steps:
            given = [self._convert(vals[i], c) for i, c in zip(ins, conv)]
            if node is None:
                vals[outs] = fn(*given)
            else:
                storage: OutputStorageType = [[None] for _ in outs]
                fn(node, given, storage)
                for k, cell in zip(outs, storage):
                    vals[k] = cell[0]
        results = [self._convert(vals[k], c) for k, c in zip(self._out_slots, self._out_conv)]
        return results[0] if self._single else results


def function(inputs: Sequence[Variable], outputs, mode=None, **_ignored) -> Function:
    """Compiles ``outputs = f(inputs)``; ``mode`` is ``"FAST_RUN"`` (default), ``"FAST_COMPILE"``
    or a :class:`Mode`.  FAST_RUN applies every rewriter tagged ``fast_run`` in position order
    (the federated ``fuse_asyncs`` pass registers itself there at position 90)."""
    single = isinstance(outputs, Variable)
    outs = [outputs] if single else list(outputs)
    fgraph = FunctionGraph(list(inputs), outs, clone=True)
    m = get_mode(mode)
    for rewriter in optdb.query(MODES.get(m.name, "fast_run"), exclude=m._excluding):
        rewriter.rewrite(fgraph)
    return Function(fgraph, single)


class FromFunctionOp(Op):
    """Wraps a Python function ``fn(*arrays) -> array(s)`` as an Op with declared types."""

    def __init__(self, fn: Callable, itypes: Sequence[Type], otypes: Sequence[Type], infer_shape=None) -> None:
        self.__fn = fn
        self.itypes = list(itypes)
        self.otypes = list(otypes)
        self.__infer_shape = infer_shape

    def make_node(self, *inputs) -> Apply:
        if len(inputs) != len(self.itypes):
            raise ValueError(f"Expected {len(self.itypes)} inputs, got {len(inputs)}")
        ins = [as_tensor(i) for i in inputs]
        for i, (var, t) in enumerate(zip(ins, self.itypes)):
            if isinstance(t, TensorType) and var.type.ndim != t.ndim:
                raise TypeError(f"Input {i} has {var.type.ndim} dimensions, expected {t.ndim}")
        return Apply(self, ins, [t() for t in self.otypes])

    def perform(self, node, inputs, output_storage) -> None:
        outs = self.__fn(*inputs)
        if not isinstance(outs, (list, tuple)):
            outs = (outs,)
        assert len(outs) == len(output_storage)
        for cell, value in zip(output_storage, outs):
            cell[0] = value
