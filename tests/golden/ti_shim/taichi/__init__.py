"""A pure-Python stand-in for the slice of Taichi that erizmr/SPH_Taichi uses (TEST INFRASTRUCTURE).

Purpose: execute the reference's OWN source files (particle_system.py, sph_base.py, WCSPH.py, DFSPH.py, imported
unmodified from a reference checkout) without the Taichi wheel, so that golden vectors for the CPU oracle come from the
reference's code rather than from a restatement of it (tests/golden/make_reference_golden.py).

Semantics implemented (what the reference relies on):
  * kernels / funcs run serially in index order -- one of the executions a parallel backend may produce; atomics
    are then plain read-modify-writes, so the counting sort is the stable one;
  * default precision: fields and vectors are float32 / int32, every arithmetic result is rounded to float32
    (numpy scalar semantics; Python-float constants act as weakly typed, as Taichi's compile-time constants do);
  * field reads yield copies, `field[i][k] = v` and `field[i].fill(v)` write through, `ti.template()` arguments
    are references (a scalar local handed to `for_all_neighbors` is boxed for the call and read back after it);
    these three are done by a small AST rewrite of each kernel / func at first call;
  * neighbour cells outside the grid are reported (counter `oob_reads`) and read as empty; golden runs assert
    that the counter stays 0, i.e. that the reference was well-defined on them.
Not implemented: anything GPU-specific (simt intrinsics exist only as names), GGUI, PLY writers, fast-math.
"""
import ast
import inspect
import itertools
import textwrap
import types as _pytypes

import numpy as np

f32 = np.float32
i32 = np.int32
f64 = np.float64
cuda, vulkan, cpu, gpu = "cuda", "vulkan", "cpu", "gpu"
oob_reads = 0


def init(*a, **k):
    pass


def data_oriented(cls):
    return cls


def _dt(t):
    if t in (float, f32, "f32"):
        return np.float32
    if t in (int, i32, "i32"):
        return np.int32
    return t


# ---- values ---------------------------------------------------------------------------------------------
class Vector:
    """Small dense vector with float32 (or int32) components and Taichi's element-wise arithmetic."""
    __array_priority__ = 100
    __array_ufunc__ = None  # numpy scalars defer to __rmul__ & co instead of building object arrays

    def __init__(self, data, dt=None):
        if isinstance(data, Vector):
            data = data.a
        a = np.array(data)
        if dt is not None:
            a = a.astype(_dt(dt))
        elif a.dtype.kind == "f":
            a = a.astype(np.float32)
        elif a.dtype.kind in "iub":
            a = a.astype(np.int32)
        self.a = a

    @staticmethod
    def zero(dt, n):
        return Vector(np.zeros(n, dtype=_dt(dt)))

    # field factory: ti.Vector.field(n, dtype, shape)
    @staticmethod
    def field(n, dtype=float, shape=None):
        return Field(_dt(dtype), shape, n)

    def _w(self, r):
        return Vector(r) if isinstance(r, np.ndarray) else r

    def _o(self, o):
        return o.a if isinstance(o, Vector) else o

    def __add__(self, o): return Vector(self.a + self._o(o))
    def __radd__(self, o): return Vector(self._o(o) + self.a)
    def __sub__(self, o): return Vector(self.a - self._o(o))
    def __rsub__(self, o): return Vector(self._o(o) - self.a)
    def __mul__(self, o): return Vector(self.a * self._o(o))
    def __rmul__(self, o): return Vector(self._o(o) * self.a)
    def __truediv__(self, o): return Vector(self.a / self._o(o))
    def __neg__(self): return Vector(-self.a)

    def __iadd__(self, o):
        self.a = (self.a + self._o(o)).astype(self.a.dtype)
        return self

    def __isub__(self, o):
        self.a = (self.a - self._o(o)).astype(self.a.dtype)
        return self

    def __imul__(self, o):
        self.a = (self.a * self._o(o)).astype(self.a.dtype)
        return self

    def __itruediv__(self, o):
        self.a = (self.a / self._o(o)).astype(self.a.dtype)
        return self

    def __getitem__(self, k): return self.a[k]
    def __setitem__(self, k, v): self.a[k] = v
    def __len__(self): return len(self.a)
    def __iter__(self): return iter(self.a)

    def cast(self, t):
        return Vector(np.trunc(self.a).astype(np.int32) if t is int else self.a.astype(_dt(t)))

    def dot(self, o):
        s = self.a[0] * o.a[0]
        for k in range(1, len(self.a)):
            s = s + self.a[k] * o.a[k]
        return s

    def norm_sqr(self):
        return self.dot(self)

    def norm(self):
        return np.sqrt(self.norm_sqr())

    def outer_product(self, o):
        return Matrix(np.outer(self.a, o.a).astype(np.float32))

    def fill(self, v):
        self.a[...] = v

    def to_numpy(self):
        return self.a.copy()

    def __repr__(self):
        return f"Vector({self.a})"


class Matrix:
    __array_priority__ = 100
    __array_ufunc__ = None

    def __init__(self, rows):
        self.a = np.array(rows.a if isinstance(rows, Matrix) else rows, dtype=np.float32)

    @staticmethod
    def identity(dt, n):
        return Matrix(np.eye(n, dtype=np.float32))

    def __add__(self, o): return Matrix(self.a + (o.a if isinstance(o, Matrix) else o))
    def __iadd__(self, o):
        self.a = (self.a + (o.a if isinstance(o, Matrix) else o)).astype(np.float32)
        return self
    def __mul__(self, o): return Matrix(self.a * (o.a if isinstance(o, Matrix) else o))
    def __rmul__(self, o): return Matrix((o.a if isinstance(o, Matrix) else o) * self.a)
    def __matmul__(self, o):
        if isinstance(o, Vector):
            return Vector((self.a @ o.a).astype(np.float32))
        return Matrix(self.a @ o.a)
    def __abs__(self): return Matrix(np.abs(self.a))
    def __lt__(self, o): return list((self.a < o).reshape(-1))  # `all(abs(R) < eps)`
    def to_numpy(self): return self.a.copy()


class Struct:
    def __init__(self, **kw):
        for k, v in kw.items():
            if isinstance(v, float):
                v = np.float32(v)
            elif isinstance(v, int) and not isinstance(v, bool):
                v = np.int32(v)
            setattr(self, k, v)


class Idx(tuple):
    """A grouped loop index: usable as a field index, and `I[0]` is the integer."""
    __slots__ = ()


class IntRef(int):
    """An int read from a field that remembers where it came from (target of ti.atomic_add / atomic_sub)."""
    def __new__(cls, value, field, index):
        obj = int.__new__(cls, value)
        obj.field, obj.index = field, index
        return obj


class Field:
    def __init__(self, dtype, shape, n=0):
        self.dtype, self.n = _dt(dtype), n
        if shape is None or shape == ():
            self.shape = ()
        elif isinstance(shape, (int, np.integer)):
            self.shape = (int(shape),)
        else:
            self.shape = tuple(int(s) for s in shape)
        self.data = np.zeros(self.shape + ((n,) if n else ()), dtype=self.dtype)

    def _ix(self, key):
        if key is None or self.shape == ():
            return ()
        if isinstance(key, tuple):
            key = key[0]
        return int(key)

    def _oob(self, ix):
        return ix != () and not (0 <= ix < self.shape[0])

    def __getitem__(self, key):
        global oob_reads
        ix = self._ix(key)
        if self._oob(ix):  # unchecked neighbour cell of the reference (SURVEY Q3): count it, read "empty"
            oob_reads += 1
            return Vector(np.zeros(self.n, self.dtype)) if self.n else self.dtype(0)
        if self.n:
            return Vector(self.data[ix].copy())
        v = self.data[ix]
        if self.dtype == np.int32:
            return IntRef(int(v), self, ix)
        return v  # numpy float32 scalar

    def __setitem__(self, key, value):
        ix = self._ix(key)
        if self.n:
            self.data[ix] = value.a if isinstance(value, (Vector,)) else value
        else:
            self.data[ix] = value

    def fill(self, v):
        self.data[...] = v

    def to_numpy(self):
        return self.data.copy()

    def from_numpy(self, a):
        self.data[...] = a


def field(dtype, shape=None):
    return Field(dtype, shape)


# ---- loops, maths, atomics ------------------------------------------------------------------------------
def grouped(x):
    if isinstance(x, Field):
        return (Idx((k,)) for k in range(x.shape[0]))
    return (Vector(np.array(t, dtype=np.int32)) for t in x)  # ti.grouped(ti.ndrange(...))


def ndrange(*ranges):
    return itertools.product(*[range(*r) if isinstance(r, tuple) else range(r) for r in ranges])


def static(x):
    return x


def loop_config(**k):
    pass


def cast(v, t):
    if isinstance(v, Vector):
        return v.cast(t)
    return _dt(t)(np.trunc(v)) if _dt(t) is np.int32 else _dt(t)(v)


def _val(v):
    return v


def max(a, b):  # noqa: A001 - mirrors ti.max
    return a if a >= b else b


def min(a, b):  # noqa: A001
    return a if a <= b else b


def abs(a):  # noqa: A001
    return Matrix.__abs__(a) if isinstance(a, Matrix) else np.abs(a)


def pow(a, b):  # noqa: A001
    return np.power(np.float32(a), np.float32(b))


def sqrt(a):
    return np.sqrt(np.float32(a))


def atomic_add(ref, v):
    old = ref.field.data[ref.index]
    ref.field.data[ref.index] = old + v
    return int(old)


def atomic_sub(ref, v):
    old = ref.field.data[ref.index]
    ref.field.data[ref.index] = old - v
    return int(old)


def polar_decompose(A):
    u, s, vt = np.linalg.svd(A.a.astype(np.float64))
    r = u @ vt
    if np.linalg.det(r) < 0:  # keep S symmetric positive semi-definite with R a rotation, as Taichi's SVD-based routine
        u[:, -1] *= -1
        s[-1] *= -1
        r = u @ vt
    sm = vt.T @ np.diag(s) @ vt
    return Matrix(r.astype(np.float32)), Matrix(sm.astype(np.float32))


def global_thread_idx():
    return 0


def template():
    return "template"


class _NS:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _unsupported(*a, **k):
    raise NotImplementedError("GPU-only intrinsic; the shim replaces the reference's scan with an exact cumsum")


simt = _NS(warp=_NS(shfl_up_i32=_unsupported, active_mask=_unsupported),
           block=_NS(sync=_unsupported), subgroup=_NS(inclusive_add=_unsupported, barrier=_unsupported))
types = _NS(ndarray=lambda *a, **k: "ndarray", vector=lambda *a, **k: "vector", matrix=lambda *a, **k: "matrix")
cfg = _NS(arch=cuda)
math = _NS(vec3=lambda *a: Vector(list(a)))


class _PrefixSumExecutor:
    """ti.algorithms.PrefixSumExecutor: in-place inclusive scan (integer-exact, any correct scan matches)."""
    def __init__(self, n):
        self.n = n

    def run(self, f):
        f.data[...] = np.cumsum(f.data, dtype=np.int64).astype(np.int32)


algorithms = _NS(PrefixSumExecutor=_PrefixSumExecutor)


# ---- the AST rewrite behind @ti.kernel / @ti.func ---------------------------------------------------------
def _box(v):
    if isinstance(v, (Vector, Matrix, Struct, np.ndarray)):
        return v
    return np.array(v, dtype=np.float32)  # 0-d array: `ret += x` inside the callee mutates it in place


def _unbox(v):
    if isinstance(v, np.ndarray) and v.shape == ():
        return np.float32(v)
    return v


def _set_comp(f, idx, k, value, op=None):
    ix = f._ix(idx)
    if op is None:
        f.data[ix][k] = value
    elif op == "add":
        f.data[ix][k] += value
    elif op == "sub":
        f.data[ix][k] -= value
    else:
        raise NotImplementedError(op)


def _fill(f, idx, value):
    f.data[f._ix(idx)][...] = value


class _Rewrite(ast.NodeTransformer):
    """field[i][k] = v  ->  ti._set_comp(field, i, k, v);   field[i].fill(v)  ->  ti._fill(field, i, v);
    `obj.for_all_neighbors(p, task, name)`  ->  box `name` before the call, unbox it after."""

    def visit_Assign(self, node):
        self.generic_visit(node)
        t = node.targets[0]
        if len(node.targets) == 1 and isinstance(t, ast.Subscript) and isinstance(t.value, ast.Subscript):
            call = ast.Call(func=ast.Attribute(value=ast.Name(id="ti", ctx=ast.Load()), attr="_set_comp", ctx=ast.Load()),
                            args=[t.value.value, t.value.slice, t.slice, node.value], keywords=[])
            return ast.copy_location(ast.Expr(value=call), node)
        return node

    def visit_Expr(self, node):
        self.generic_visit(node)
        c = node.value
        if isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute):
            if c.func.attr == "fill" and isinstance(c.func.value, ast.Subscript):
                call = ast.Call(func=ast.Attribute(value=ast.Name(id="ti", ctx=ast.Load()), attr="_fill", ctx=ast.Load()),
                                args=[c.func.value.value, c.func.value.slice, c.args[0]], keywords=[])
                return ast.copy_location(ast.Expr(value=call), node)
            if c.func.attr == "for_all_neighbors" and len(c.args) == 3 and isinstance(c.args[2], ast.Name):
                name = c.args[2].id
                def mk(fn):
                    return ast.Assign(targets=[ast.Name(id=name, ctx=ast.Store())],
                                      value=ast.Call(func=ast.Attribute(value=ast.Name(id="ti", ctx=ast.Load()), attr=fn, ctx=ast.Load()),
                                                     args=[ast.Name(id=name, ctx=ast.Load())], keywords=[]))
                return [ast.copy_location(mk("_box"), node), node, ast.copy_location(mk("_unbox"), node)]
        return node


def _compile(fn):
    src = textwrap.dedent(inspect.getsource(fn))
    tree = ast.parse(src)
    fdef = tree.body[0]
    fdef.decorator_list = []
    for a in fdef.args.args:  # annotations like ti.types.ndarray() are irrelevant here
        a.annotation = None
    fdef.returns = None
    tree = ast.fix_missing_locations(_Rewrite().visit(tree))
    glb = fn.__globals__
    glb.setdefault("ti", __import__(__name__))
    loc = {}
    exec(compile(tree, inspect.getsourcefile(fn) or "<ti-shim>", "exec"), glb, loc)
    return loc[fdef.name]


def _decorate(fn):
    cache = {}

    def wrapper(*a, **k):
        if "f" not in cache:
            cache["f"] = _compile(fn)
        return cache["f"](*a, **k)

    wrapper.__name__ = getattr(fn, "__name__", "ti_fn")
    wrapper.__wrapped__ = fn

    class _Desc:  # behaves as a plain function on modules and as a method on classes
        def __get__(self, obj, objtype=None):
            if obj is None:
                return wrapper
            return _pytypes.MethodType(wrapper, obj)

        def __call__(self, *a, **k):
            return wrapper(*a, **k)

    return _Desc()


kernel = _decorate
func = _decorate
