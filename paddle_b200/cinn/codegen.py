"""Code generation for a fusion group: CUDA C++ for sm_90a (the product) and plain C++ for the host (how the compiler is exercised on a
machine without a GPU; same expression bodies).

Schedules
  * elementwise group  -> one grid-stride kernel over the flat domain; a second variant moves 4 elements per thread (8 when a 16-bit tensor is
    streamed, so that its accesses are 16 bytes wide; picked at launch when every pointer is 16-byte aligned); the grid is capped at 132 SMs x 8 CTAs.
  * group with reductions over the last axis -> a row kernel: one warp per row for rows of <= 256 columns (shuffle reductions, 8 rows per
    CTA), one 256-thread CTA per row up to 2048 columns, one 1024-thread CTA per row beyond (shuffle + one shared-memory exchange).
    Reductions that feed later elementwise work become successive passes over the row (pass s computes every reduction whose input depends
    on s earlier reductions).  Up to 8192 columns every thread owns <= 8 columns, the column loops are unrolled over them and a value a
    later pass reads again stays in a register array (softmax numerator, centred input of a normalisation); longer rows recompute from the
    inputs through L1 / L2.  Per-row values live in registers; the per-row part of every broadcast index is hoisted out of the column loops.
  * group with sums over LEADING axes (bias gradients, batch statistics) -> the domain is read as [A, K, B]; CTAs of 32 columns x 8 k-lanes, the K
    range split over `split` CTAs that leave fp32 partials, a second kernel adds them (deterministic, no atomics).
Role parity: CINN's group schedule + CodeGenCUDA_Dev (paddle/cinn/ir/group_schedule, paddle/cinn/backends/codegen_cuda_dev.cc)."""
from __future__ import annotations

import math

from .expr import COMPARE, Node, Unsupported, compute_type

_RANK = {"bool": 0, "int": 1, "long long": 2, "float": 3, "double": 4}
_STORE = {"float32": "float", "float64": "double", "float16": "__half", "bfloat16": "__nv_bfloat16", "int32": "int", "int64": "long long", "bool": "bool", "uint8": "unsigned char"}
_ESIZE = {"float32": 4, "float64": 8, "float16": 2, "bfloat16": 2, "int32": 4, "int64": 8, "bool": 1, "uint8": 1}


def _prod(xs):
    p = 1
    for x in xs:
        p *= int(x)
    return p


def _lit(v, cty):
    if cty == "bool":
        return "true" if v else "false"
    if cty in ("int", "long long"):
        if isinstance(v, float) and not float(v).is_integer():
            raise Unsupported("fractional literal in an integer expression")
        return f"{int(v)}" + ("LL" if cty == "long long" else "")
    v = float(v)
    if math.isnan(v):
        return "NAN" if cty == "float" else "(double)NAN"
    if math.isinf(v):
        s = "INFINITY" if v > 0 else "-INFINITY"
        return s if cty == "float" else f"(double)({s})"
    r = repr(v)
    if "e" not in r and "." not in r:
        r += ".0"
    return r + ("f" if cty == "float" else "")


def _promote(ctys):
    return max(ctys, key=lambda c: _RANK[c])


class Spec:
    """What codegen needs: the domain, the nodes (topological), the input nodes in operand order, the output nodes in result order."""

    def __init__(self, name, full, nodes, inputs, outputs):
        self.name, self.full, self.nodes, self.inputs, self.outputs = name, tuple(full), nodes, inputs, outputs
        if len({id(n) for n in outputs}) != len(outputs):
            raise ValueError("a group result is listed twice")
        self.cols = int(full[-1]) if full else 1
        self.rows = _prod(full[:-1]) if full else 1
        # row schedule: reductions, or per-row values (e.g. the gradient of a non-keepdim row result on its way back to the columns)
        self.has_reduce = any(n.kind == "reduce" or (n.kind == "ew" and n.space == "row") for n in nodes)
        self.col = [n for n in nodes if n.kind == "creduce"]            # column reductions: the group runs on the [A, K, B] schedule
        self.akb = self.col[0].attrs["akb"] if self.col else None
        for n in nodes:                                   # levels: how many reductions deep a value is
            if n.kind == "in":
                n.level = 0
            elif n.kind == "reduce":
                n.level = n.args[0].level + 1
            else:
                n.level = max([a.level for a in n.args if isinstance(a, Node)] or [0])
        self.max_level = max([n.level for n in nodes if n.kind == "reduce"] or [0])


class _Body:
    """Emits C statements for nodes.  `names[(node id, context)]` is the variable that holds a node's value in a context ('full' inside a
    column loop, 'row' per row)."""

    def __init__(self, spec):
        self.spec = spec
        self.lead = spec.full[:-1]

    def cty(self, n):
        return compute_type(n.dtype)

    # ---- broadcast index of an input read in a context --------------------------------------------------------------------------------
    def in_index(self, n, ctx):
        """(row part as a C expression in `row` or None when it is 0, uses_j).  Inputs are contiguous."""
        shape = tuple(n.shape)
        lead = self.lead
        if ctx == "full":
            target = self.spec.full
        else:
            target = lead          # row contexts: the flat index IS `row`
            if ctx == "keep":      # consumer is S[:-1] + (1,): the input's last axis lines up with that 1 and carries no stride
                if shape:
                    if shape[-1] != 1:
                        raise Unsupported(f"cannot broadcast {list(n.shape)} per row")
                    shape = shape[:-1]
        if len(shape) > len(target):
            if all(d == 1 for d in shape[: len(shape) - len(target)]):
                shape = shape[len(shape) - len(target):]
            else:
                raise Unsupported("input rank exceeds its context")
        padded = (1,) * (len(target) - len(shape)) + shape
        for a, b in zip(padded, target):
            if a != 1 and a != b:
                raise Unsupported(f"cannot broadcast {list(n.shape)}")
        if ctx == "full" and target:
            uses_j = padded[-1] != 1
            lead_in, last_stride = padded[:-1], (padded[-1] if padded else 1)
        else:
            uses_j, lead_in, last_stride = False, padded, 1
        # collapse runs of leading dims with the same broadcast status; row = sum_g idx_g * prod(lead[after g])
        terms, d, nl = [], 0, len(lead)
        while d < nl:
            e = d
            bc = lead_in[d] == 1 and lead[d] != 1
            while e < nl and ((lead_in[e] == 1 and lead[e] != 1) == bc or lead[e] == 1):
                e += 1
            if not bc:
                size, after = _prod(lead[d:e]), _prod(lead[e:])
                stride = _prod(lead_in[e:]) * last_stride
                if size > 1:
                    idx = "row" if after == 1 else f"(row / {after}LL)"
                    if d > 0 and _prod(lead[:d]) > 1:
                        idx = f"({idx} % {size}LL)"
                    terms.append(idx if stride == 1 else f"{idx} * {stride}LL")
            d = e
        return (" + ".join(terms) if terms else None), uses_j

    # ---- one elementwise node ------------------------------------------------------------------------------------------------------------
    def ew_expr(self, n, ref):
        """C expression of an `ew` node; `ref(arg)` gives (expression, C type) of a Node argument."""
        T = self.cty(n)
        f = T in ("float", "double")
        sfx = "f" if T == "float" else ""

        def val(a, to):
            if isinstance(a, Node):
                e, t = ref(a)
                return e if t == to else f"(({to}){e})"
            return _lit(a, to)

        op, args = n.op, n.args
        if op == "cast":
            return val(args[0], T)
        if op == "where":
            return f"({val(args[0], 'bool')} ? {val(args[1], T)} : {val(args[2], T)})"
        if op in COMPARE:
            ts = [ref(a)[1] if isinstance(a, Node) else ("float" if isinstance(a, float) else "int") for a in args]
            P = _promote(ts)
            sym = {"gt": ">", "lt": "<", "ge": ">=", "le": "<=", "eq": "==", "ne": "!="}[op]
            return f"({val(args[0], P)} {sym} {val(args[1], P)})"
        if op in ("logical_and", "logical_or"):
            return f"({val(args[0], 'bool')} {'&&' if op == 'logical_and' else '||'} {val(args[1], 'bool')})"
        if op == "logical_not":
            return f"(!{val(args[0], 'bool')})"
        if T == "bool":
            raise Unsupported(f"{op} on bool")
        a = val(args[0], T)
        b = val(args[1], T) if len(args) > 1 else None
        if op in ("add", "sub", "mul"):
            return f"({a} {dict(add='+', sub='-', mul='*')[op]} {b})"
        if op == "div":
            if not f:
                raise Unsupported("integer true division")
            return f"({a} / {b})"
        if op == "floordiv":
            return f"floor{sfx}({a} / {b})" if f else f"cinn_floordiv({a}, {b})"
        if op == "fmod":
            return f"fmod{sfx}({a}, {b})" if f else f"cinn_mod({a}, {b})"
        if op == "maximum":
            return f"cinn_max({a}, {b})"
        if op == "minimum":
            return f"cinn_min({a}, {b})"
        if op == "neg":
            return f"(-{a})"
        if op == "square":
            return f"({a} * {a})"
        if op == "abs":
            return f"fabs{sfx}({a})" if f else f"({a} < 0 ? -{a} : {a})"
        if op == "relu":
            return f"({a} < {_lit(0, T)} ? {_lit(0, T)} : {a})"
        if op == "sign":
            return f"(({T})(({a} > {_lit(0, T)}) - ({a} < {_lit(0, T)})))"
        if not f:
            raise Unsupported(f"{op} on integers")
        one = _lit(1.0, T)
        if op == "pow":
            return f"pow{sfx}({a}, {b})"
        if op == "reciprocal":
            return f"({one} / {a})"
        if op == "sigmoid":
            return f"({one} / ({one} + exp{sfx}(-{a})))"
        if op == "rsqrt":
            return f"({one} / sqrt{sfx}({a}))"
        if op == "round":
            return f"nearbyint{sfx}({a})"
        fn = {"exp": "exp", "log": "log", "sqrt": "sqrt", "tanh": "tanh", "erf": "erf", "sin": "sin", "cos": "cos", "floor": "floor", "ceil": "ceil", "log1p": "log1p",
              "expm1": "expm1", "exp2": "exp2"}.get(op)
        if fn is None:
            raise Unsupported(f"no code for {op}")
        return f"{fn}{sfx}({a})"


_RED_INIT = {"sum": lambda T: _lit(0, T), "max": lambda T: _lit(float("-inf"), T), "min": lambda T: _lit(float("inf"), T)}
_RED_COMB = {"sum": "({a} + {b})", "max": "cinn_max({a}, {b})", "min": "cinn_min({a}, {b})"}
_RED_ID = {"sum": 0, "max": 1, "min": 2}

_COMMON = r"""
template <class T> CINN_HD inline T cinn_max(T a, T b) { return (a != a || a > b) ? a : b; }     // NaN propagates, as in the eager ops
template <class T> CINN_HD inline T cinn_min(T a, T b) { return (a != a || a < b) ? a : b; }
template <class T> CINN_HD inline T cinn_floordiv(T a, T b) {        // integers; a zero divisor yields -1 (what the device does) instead of trapping the host
  if (b == 0) return (T)-1;
  T q = a / b;
  return ((a % b != 0) && ((a < 0) != (b < 0))) ? q - 1 : q;
}
template <class T> CINN_HD inline T cinn_mod(T a, T b) { return b == 0 ? (T)-1 : a % b; }
template <class T> CINN_HD inline T cinn_comb(int op, T a, T b) { return op == 0 ? a + b : (op == 1 ? cinn_max(a, b) : cinn_min(a, b)); }
"""

_CUDA_PRELUDE = r"""
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <math.h>
#define CINN_HD __host__ __device__
""" + _COMMON + r"""
__device__ inline float ld(const float* p, long long i) { return p[i]; }
__device__ inline double ld(const double* p, long long i) { return p[i]; }
__device__ inline float ld(const __half* p, long long i) { return __half2float(p[i]); }
__device__ inline float ld(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
__device__ inline int ld(const int* p, long long i) { return p[i]; }
__device__ inline long long ld(const long long* p, long long i) { return p[i]; }
__device__ inline bool ld(const bool* p, long long i) { return p[i]; }
__device__ inline int ld(const unsigned char* p, long long i) { return p[i]; }
__device__ inline void st(float* p, long long i, float v) { p[i] = v; }
__device__ inline void st(double* p, long long i, double v) { p[i] = v; }
__device__ inline void st(__half* p, long long i, float v) { p[i] = __float2half_rn(v); }
__device__ inline void st(__nv_bfloat16* p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }
__device__ inline void st(int* p, long long i, int v) { p[i] = v; }
__device__ inline void st(long long* p, long long i, long long v) { p[i] = v; }
__device__ inline void st(bool* p, long long i, bool v) { p[i] = v; }
__device__ inline void st(unsigned char* p, long long i, int v) { p[i] = (unsigned char)v; }
// V consecutive elements per access: raw 16 / 8 / 4-byte chunks, converted element by element in registers
template <int V, class S> struct __align__((V * sizeof(S)) >= 16 ? 16 : (V * sizeof(S))) CinnRaw { S e[V]; };
template <int V, class S> __device__ inline void cinn_ld_raw(CinnRaw<V, S>& r, const S* p) {
  constexpr int B = V * sizeof(S);
  if constexpr (B % 16 == 0) {
#pragma unroll
    for (int k = 0; k < B / 16; ++k) reinterpret_cast<uint4*>(&r)[k] = reinterpret_cast<const uint4*>(p)[k];
  } else if constexpr (B == 8) {
    *reinterpret_cast<uint2*>(&r) = *reinterpret_cast<const uint2*>(p);
  } else {
    static_assert(B == 4, "vector access of 4, 8 or a multiple of 16 bytes");
    *reinterpret_cast<unsigned*>(&r) = *reinterpret_cast<const unsigned*>(p);
  }
}
template <int V, class S> __device__ inline void cinn_st_raw(const CinnRaw<V, S>& r, S* p) {
  constexpr int B = V * sizeof(S);
  if constexpr (B % 16 == 0) {
#pragma unroll
    for (int k = 0; k < B / 16; ++k) reinterpret_cast<uint4*>(p)[k] = reinterpret_cast<const uint4*>(&r)[k];
  } else if constexpr (B == 8) {
    *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(&r);
  } else {
    *reinterpret_cast<unsigned*>(p) = *reinterpret_cast<const unsigned*>(&r);
  }
}
template <int V, class S, class T> __device__ inline void ldv(const S* p, long long i, T (&o)[V]) {
  CinnRaw<V, S> r;
  cinn_ld_raw<V, S>(r, p + i);
#pragma unroll
  for (int u = 0; u < V; ++u) o[u] = ld(&r.e[u], 0);
}
template <int V, class S, class T> __device__ inline void stv(S* p, long long i, const T (&o)[V]) {
  CinnRaw<V, S> r;
#pragma unroll
  for (int u = 0; u < V; ++u) st(&r.e[u], 0, o[u]);
  cinn_st_raw<V, S>(r, p + i);
}
template <class T> __device__ inline T cinn_warp_reduce(int op, T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = cinn_comb(op, v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <class T> __device__ inline T cinn_block_reduce(int op, T v, T identity, void* smem) {
  T* buf = reinterpret_cast<T*>(smem);
  v = cinn_warp_reduce(op, v);
  __syncthreads();                                   // the previous reduction's readers are done with the buffer
  if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
  __syncthreads();
  v = threadIdx.x < (blockDim.x >> 5) ? buf[threadIdx.x] : identity;
  if (threadIdx.x < 32) v = cinn_warp_reduce(op, v);
  if (threadIdx.x == 0) buf[0] = v;
  __syncthreads();
  return buf[0];
}
"""

_HOST_PRELUDE = r"""
#include <math.h>
#include <stdint.h>
#include <string.h>
#define CINN_HD
""" + _COMMON + r"""
struct __half { uint16_t x; };
struct __nv_bfloat16 { uint16_t x; };
static inline float bf2f(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; memcpy(&f, &u, 4); return f; }
static inline uint16_t f2bf(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);      // NaN stays NaN
  u += 0x7fffu + ((u >> 16) & 1u);                                               // round to nearest even
  return (uint16_t)(u >> 16);
}
static inline float h2f(uint16_t h) { _Float16 v; memcpy(&v, &h, 2); return (float)v; }
static inline uint16_t f2h(float f) { _Float16 v = (_Float16)f; uint16_t h; memcpy(&h, &v, 2); return h; }
static inline float ld(const float* p, long long i) { return p[i]; }
static inline double ld(const double* p, long long i) { return p[i]; }
static inline float ld(const __half* p, long long i) { return h2f(p[i].x); }
static inline float ld(const __nv_bfloat16* p, long long i) { return bf2f(p[i].x); }
static inline int ld(const int* p, long long i) { return p[i]; }
static inline long long ld(const long long* p, long long i) { return p[i]; }
static inline bool ld(const bool* p, long long i) { return p[i]; }
static inline int ld(const unsigned char* p, long long i) { return p[i]; }
static inline void st(float* p, long long i, float v) { p[i] = v; }
static inline void st(double* p, long long i, double v) { p[i] = v; }
static inline void st(__half* p, long long i, float v) { p[i].x = f2h(v); }
static inline void st(__nv_bfloat16* p, long long i, float v) { p[i].x = f2bf(v); }
static inline void st(int* p, long long i, int v) { p[i] = v; }
static inline void st(long long* p, long long i, long long v) { p[i] = v; }
static inline void st(bool* p, long long i, bool v) { p[i] = v; }
static inline void st(unsigned char* p, long long i, int v) { p[i] = (unsigned char)v; }
"""


class _Plan:
    """Which nodes each loop computes (shared by both targets)."""

    def __init__(self, spec):
        self.spec = spec
        nodes = spec.nodes
        self.stage_reduces = {s: [n for n in nodes if n.kind == "reduce" and n.level == s + 1] for s in range(spec.max_level)}
        self.row_ews = {s: [n for n in nodes if n.kind == "ew" and n.space == "row" and n.level == s] for s in range(spec.max_level + 1)}
        self.full_outputs = [n for n in spec.outputs if n.kind == "ew" and n.space == "full"]
        self.row_outputs = [n for n in spec.outputs if n.space == "row"]

    def full_closure(self, targets):
        """Full-space nodes (and inputs read per element) a column loop has to evaluate for `targets`, in topological order."""
        need, stack = set(), [t.args[0] if t.kind == "creduce" else t for t in targets]
        while stack:
            n = stack.pop()
            if n.id in need:
                continue
            if n.kind == "in" or (n.kind == "ew" and n.space == "full"):
                need.add(n.id)
                if n.kind == "ew":
                    stack.extend(a for a in n.args if isinstance(a, Node))
        return [n for n in self.spec.nodes if n.id in need]


def _params(spec):
    ps = [f"const {_STORE[n.dtype]}* __restrict__ in{k}" for k, n in enumerate(spec.inputs)]
    ps += [f"{_STORE[n.dtype]}* __restrict__ out{k}" for k, n in enumerate(spec.outputs)]
    return ", ".join(ps + ["long long rows"])


def _call_args(spec):
    a = [f"(const {_STORE[n.dtype]}*)in[{k}]" for k, n in enumerate(spec.inputs)]
    a += [f"({_STORE[n.dtype]}*)out[{k}]" for k, n in enumerate(spec.outputs)]
    return ", ".join(a + ["rows"])


class _RowEmitter:
    """Statements of the row schedule, parametrised by how a column loop and a reduction are written.

    `cache_per` (CUDA, short rows): every thread owns at most `cache_per` columns of the row, the column loops are fully unrolled over them and
    a value that a LATER loop reads again (the softmax numerator, the centred input of a normalisation, ...) is kept in a register array
    instead of being recomputed from global memory.  Without it (host, long rows) later loops recompute from the inputs."""

    def __init__(self, spec, loop_open, reduce_stmt, indent="    ", cache_per=None, loop_close="}"):
        self.spec, self.body, self.plan = spec, _Body(spec), _Plan(spec)
        self.loop_open, self.loop_close, self.reduce_stmt, self.ind = loop_open, loop_close, reduce_stmt, indent
        self.in_pos = {n.id: k for k, n in enumerate(spec.inputs)}
        self.out_pos = {n.id: k for k, n in enumerate(spec.outputs)}
        self.lines = []
        self.row_named = {}              # node id -> per-row variable
        self.hoisted = set()
        self.cache_per = cache_per
        self.loops = self._plan_loops()

    def w(self, s, extra=0):
        self.lines.append(self.ind + "  " * extra + s)

    # ---- which loop computes what ----------------------------------------------------------------------------------------------------------
    def _loop_targets(self):
        spec, plan = self.spec, self.plan
        t = [[r.args[0] for r in plan.stage_reduces[s]] for s in range(spec.max_level)]
        if plan.full_outputs:
            t.append(list(plan.full_outputs))
        return t

    def _per_element(self, n):
        """Is this node evaluated per column?  (full-space ew nodes, inputs whose index moves with the column)"""
        return (n.kind == "ew" and n.space == "full") or (n.kind == "in" and self.body.in_index(n, "full")[1])

    def _plan_loops(self):
        """[(nodes computed in the loop, nodes read from the register cache)] per column loop; sets self.cached."""
        by_id = {n.id: n for n in self.spec.nodes}
        targets = self._loop_targets()
        if self.cache_per is None:
            self.cached = set()
            return [([by_id[n.id] for n in self.plan.full_closure(t)], []) for t in targets]
        home, cached, loops = {}, set(), []
        for i, t in enumerate(targets):
            need, reads, stack = set(), set(), list(t)
            while stack:
                n = stack.pop()
                if n.id in need or n.id in reads:
                    continue
                if n.kind == "in" or (n.kind == "ew" and n.space == "full"):
                    if n.id in home and self._per_element(n):
                        reads.add(n.id)
                        continue
                    need.add(n.id)
                    if n.kind == "ew":
                        stack.extend(a for a in n.args if isinstance(a, Node))
            for nid in need:
                home.setdefault(nid, i)
            cached |= reads
            loops.append(([n for n in self.spec.nodes if n.id in need], [n for n in self.spec.nodes if n.id in reads]))
        if len(cached) * self.cache_per > 64:          # too many live registers: recompute instead
            self.cache_per = None
            return self._plan_loops()
        self.cached = cached
        return loops

    def _hoist_input(self, n, ctx):
        """Per-row part of an input's index (and the whole load when the column does not enter)."""
        key = (n.id, ctx)
        if key in self.hoisted:
            return
        self.hoisted.add(key)
        rowpart, uses_j = self.body.in_index(n, ctx)
        k = self.in_pos[n.id]
        if uses_j:
            self.w(f"const long long ro{n.id} = {rowpart or '0'};")
        else:
            self.w(f"const {compute_type(n.dtype)} r{n.id}_{ctx[0]} = ld(in{k}, {rowpart or '0'});")

    def _ref_full(self, a):
        if a.kind == "in":
            _, uses_j = self.body.in_index(a, "full")
            return (f"v{a.id}" if uses_j else f"r{a.id}_f"), compute_type(a.dtype)
        if a.space == "row":
            return self.row_named[a.id], compute_type(a.dtype)
        return f"v{a.id}", compute_type(a.dtype)

    def _row_ctx(self, n):
        """Row context of a per-row node: 'keep' for S[:-1] + (1,), 'row' for S[:-1]."""
        return "keep" if len(n.shape) == len(self.spec.full) and self.spec.full else "row"

    def _ref_row_for(self, ctx):
        def ref(a):
            if a.kind == "in":
                return f"r{a.id}_{ctx[0]}", compute_type(a.dtype)
            return self.row_named[a.id], compute_type(a.dtype)

        return ref

    def column_loop(self, k, per_element):
        """for j: evaluate loop k's nodes, then the `per_element()` statements."""
        compute, reads = self.loops[k]
        for n in compute:
            if n.kind == "in":
                self._hoist_input(n, "full")
        self.w(self.loop_open)
        for n in reads:
            self.w(f"const {compute_type(n.dtype)} v{n.id} = c{n.id}[it];", 1)
        for n in compute:
            if n.kind == "in":
                if not self.body.in_index(n, "full")[1]:
                    continue
                self.w(f"const {compute_type(n.dtype)} v{n.id} = ld(in{self.in_pos[n.id]}, ro{n.id} + j);", 1)
            else:
                self.w(f"const {compute_type(n.dtype)} v{n.id} = {self.body.ew_expr(n, self._ref_full)};", 1)
            if n.id in self.cached:
                self.w(f"c{n.id}[it] = v{n.id};", 1)
        for s in per_element():
            self.w(s, 1)
        self.w(self.loop_close)

    def row_values(self, level):
        for n in self.plan.row_ews[level]:
            ctx = self._row_ctx(n)
            for a in n.args:
                if isinstance(a, Node) and a.kind == "in":
                    self._hoist_input(a, ctx)
            self.row_named[n.id] = f"r{n.id}"
            self.w(f"const {compute_type(n.dtype)} r{n.id} = {self.body.ew_expr(n, self._ref_row_for(ctx))};")

    def emit(self, store_guard=None):
        spec, plan = self.spec, self.plan
        by_id = {n.id: n for n in spec.nodes}
        for nid in sorted(self.cached):
            self.w(f"{compute_type(by_id[nid].dtype)} c{nid}[{self.cache_per}];")
        self.row_values(0)
        for s in range(spec.max_level):
            reds = plan.stage_reduces[s]
            for r in reds:
                T = compute_type(r.dtype)
                self.w(f"{T} acc{r.id} = {_RED_INIT[r.op](T)};")

            def per_element(reds=reds):
                out = []
                for r in reds:
                    T = compute_type(r.dtype)
                    x, xt = self._ref_full(r.args[0])
                    x = x if xt == T else f"(({T}){x})"
                    out.append(f"acc{r.id} = {_RED_COMB[r.op].format(a=f'acc{r.id}', b=x)};")
                return out

            self.column_loop(s, per_element)
            for r in reds:
                T = compute_type(r.dtype)
                self.w(self.reduce_stmt(r, T))
                self.row_named[r.id] = f"r{r.id}"
            self.row_values(s + 1)
        if plan.full_outputs:
            def stores():
                return [f"st(out{self.out_pos[n.id]}, row * {spec.cols}LL + j, v{n.id});" for n in plan.full_outputs]

            self.column_loop(spec.max_level, stores)
        for n in plan.row_outputs:
            stmt = f"st(out{self.out_pos[n.id]}, row, {self.row_named[n.id]});"
            self.w(f"if ({store_guard}) {stmt}" if store_guard else stmt)
        return "\n".join(self.lines)


def _col_body(spec, ld_indent):
    """Per-element statements of a column-reduction group, for `e` (flat index), `row`, `j` in scope: loads, the closure of every result, stores
    of the full results; returns (lines, names of the values the reductions add up)."""
    body = _Body(spec)
    in_pos = {n.id: k for k, n in enumerate(spec.inputs)}
    out_pos = {n.id: k for k, n in enumerate(spec.outputs)}
    closure = _Plan(spec).full_closure(spec.outputs)
    idx = {n.id: body.in_index(n, "full") for n in closure if n.kind == "in"}

    def ref(a):
        return f"v{a.id}", compute_type(a.dtype)

    L = []
    for n in closure:
        T = compute_type(n.dtype)
        if n.kind == "in":
            rp, uj = idx[n.id]
            off = "e" if tuple(n.shape) == spec.full else (" + ".join(([f"({rp})"] if rp else []) + (["j"] if uj else [])) or "0")
            L.append(f"{ld_indent}const {T} v{n.id} = ld(in{in_pos[n.id]}, {off});")
        else:
            L.append(f"{ld_indent}const {T} v{n.id} = {body.ew_expr(n, ref)};")
    for n in spec.outputs:
        if n.kind == "ew":
            L.append(f"{ld_indent}st(out{out_pos[n.id]}, e, v{n.id});")
    return L, out_pos


def _host_col_source(spec):
    A, K, B = spec.akb
    lines, out_pos = _col_body(spec, "        ")
    L = [_HOST_PRELUDE, "extern \"C\" int cinn_run(void** in, void** out, long long rows, int aux) {", "  (void)rows; (void)aux;"]
    L += [f"  const {_STORE[n.dtype]}* in{k} = (const {_STORE[n.dtype]}*)in[{k}];" for k, n in enumerate(spec.inputs)]
    L += [f"  {_STORE[n.dtype]}* out{k} = ({_STORE[n.dtype]}*)out[{k}];" for k, n in enumerate(spec.outputs)]
    L.append(f"  for (long long a = 0; a < {A}LL; ++a) for (long long b = 0; b < {B}LL; ++b) {{")
    for r in spec.col:
        L.append(f"    {compute_type(r.dtype)} acc{r.id} = 0;")
    L.append(f"    for (long long k = 0; k < {K}LL; ++k) {{")
    L.append(f"      const long long e = (a * {K}LL + k) * {B}LL + b; const long long row = e / {spec.cols}LL; const long long j = e - row * {spec.cols}LL; (void)row; (void)j;")
    L += lines
    for r in spec.col:
        L.append(f"        acc{r.id} += ({compute_type(r.dtype)})v{r.args[0].id};")
    L.append("    }")
    for r in spec.col:
        sc = r.attrs.get("scale")
        T = compute_type(r.dtype)
        L.append(f"    st(out{out_pos[r.id]}, a * {B}LL + b, acc{r.id}{'' if sc is None else ' * ' + _lit(sc, T)});")
    L.append("  }\n  return 0;\n}")
    return "\n".join(L) + "\n"


def host_source(spec):
    if spec.col:
        return _host_col_source(spec)
    em = _RowEmitter(spec, f"for (int j = 0; j < {spec.cols}; ++j) {{", lambda r, T: f"const {T} r{r.id} = acc{r.id};")
    body = em.emit()
    return (_HOST_PRELUDE + f"\nextern \"C\" int cinn_run(void** in, void** out, long long rows, int aux) {{\n  (void)aux;\n"
            + "".join(f"  const {_STORE[n.dtype]}* in{k} = (const {_STORE[n.dtype]}*)in[{k}];\n" for k, n in enumerate(spec.inputs))
            + "".join(f"  {_STORE[n.dtype]}* out{k} = ({_STORE[n.dtype]}*)out[{k}];\n" for k, n in enumerate(spec.outputs))
            + f"  for (long long row = 0; row < rows; ++row) {{\n{body}\n  }}\n  return 0;\n}}\n")


# ---- CUDA ------------------------------------------------------------------------------------------------------------------------------
SM_COUNT = 132


def _vec_width(spec):
    """Elements per thread of the vector variant: 8 when a 16-bit (or narrower) tensor is streamed (16-byte accesses for it), else 4; 0 = none."""
    body = _Body(spec)
    sizes = []
    for n in list(spec.inputs) + list(spec.outputs):
        if n.kind == "in" and not body.in_index(n, "full")[1]:
            continue                                       # read once per row, not streamed
        sizes.append(_ESIZE[n.dtype])
    if not sizes:
        return 0
    if min(sizes) <= 2 and spec.cols % 8 == 0:
        return 8
    return 4 if spec.cols % 4 == 0 else 0


def _flat_kernels(spec):
    """Elementwise group: scalar kernel + a V-wide vector kernel."""
    body = _Body(spec)
    in_pos = {n.id: k for k, n in enumerate(spec.inputs)}
    closure = _Plan(spec).full_closure(spec.outputs)
    idx = {n.id: body.in_index(n, "full") for n in closure if n.kind == "in"}
    same = {n.id: (tuple(n.shape) == spec.full) for n in closure if n.kind == "in"}
    need_rj = any(not same[i] for i in idx)

    def ref(a):
        return f"v{a.id}", compute_type(a.dtype)

    def offset(n, jvar):
        rp, uj = idx[n.id]
        if same[n.id]:
            return "e"
        parts = ([f"({rp})"] if rp else []) + ([jvar] if uj else [])
        return " + ".join(parts) if parts else "0"

    L = []
    L.append(f"extern \"C\" __global__ void __launch_bounds__(256) cinn_k_flat({_params(spec)}) {{")
    L.append(f"  const long long n = rows * {spec.cols}LL;")
    L.append("  for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n; e += gridDim.x * 256LL) {")
    if need_rj:
        L.append(f"    const long long row = e / {spec.cols}LL; const long long j = e - row * {spec.cols}LL; (void)row; (void)j;")
    for n in closure:
        T = compute_type(n.dtype)
        if n.kind == "in":
            L.append(f"    const {T} v{n.id} = ld(in{in_pos[n.id]}, {offset(n, 'j')});")
        else:
            L.append(f"    const {T} v{n.id} = {body.ew_expr(n, ref)};")
    for k, n in enumerate(spec.outputs):
        L.append(f"    st(out{k}, e, v{n.id});")
    L.append("  }\n}")
    V = _vec_width(spec)
    if V:
        L.append(f"extern \"C\" __global__ void __launch_bounds__(256) cinn_k_vec{V}({_params(spec)}) {{")
        L.append(f"  const long long ng = rows * {spec.cols // V}LL;")
        L.append("  for (long long g = blockIdx.x * 256LL + threadIdx.x; g < ng; g += gridDim.x * 256LL) {")
        L.append(f"    const long long e = g * {V}; const long long row = e / {spec.cols}LL; const long long j = e - row * {spec.cols}LL; (void)row; (void)j;")
        for n in closure:
            if n.kind == "in":
                T = compute_type(n.dtype)
                if idx[n.id][1]:
                    L.append(f"    {T} a{n.id}[{V}]; ldv<{V}>(in{in_pos[n.id]}, {offset(n, 'j')}, a{n.id});")
                else:
                    L.append(f"    const {T} s{n.id} = ld(in{in_pos[n.id]}, {offset(n, 'j')});")
        for k, n in enumerate(spec.outputs):
            L.append(f"    {compute_type(n.dtype)} o{k}[{V}];")
        L.append("#pragma unroll")
        L.append(f"    for (int u = 0; u < {V}; ++u) {{")
        for n in closure:
            T = compute_type(n.dtype)
            if n.kind == "in":
                L.append(f"      const {T} v{n.id} = {f'a{n.id}[u]' if idx[n.id][1] else f's{n.id}'};")
            else:
                L.append(f"      const {T} v{n.id} = {body.ew_expr(n, ref)};")
        for k, n in enumerate(spec.outputs):
            L.append(f"      o{k}[u] = v{n.id};")
        L.append("    }")
        for k, n in enumerate(spec.outputs):
            L.append(f"    stv<{V}>(out{k}, e, o{k});")
        L.append("  }\n}")
    return "\n".join(L)


def _row_schedule(cols):
    """(lanes per row, threads per CTA, rows per CTA, columns per thread or None)"""
    if cols <= 256:
        return 32, 256, 8, -(-cols // 32)
    if cols <= 2048:
        return 256, 256, 1, -(-cols // 256)
    if cols <= 8192:
        return 1024, 1024, 1, -(-cols // 1024)
    return 1024, 1024, 1, None


def _row_kernel(spec):
    lanes, threads, rpb, per = _row_schedule(spec.cols)
    warp = lanes == 32
    if warp:
        red = lambda r, T: f"const {T} r{r.id} = cinn_warp_reduce({_RED_ID[r.op]}, acc{r.id});"
    else:
        red = lambda r, T: f"const {T} r{r.id} = cinn_block_reduce({_RED_ID[r.op]}, acc{r.id}, {_RED_INIT[r.op](T)}, (void*)cinn_smem);"
    if per is not None:
        em = _RowEmitter(spec, f"_Pragma(\"unroll\") for (int it = 0; it < {per}; ++it) {{ const int j = lane + it * {lanes}; if (j < {spec.cols}) {{", red,
                         cache_per=per, loop_close="} }")
    if per is None or em.cache_per is None:
        em = _RowEmitter(spec, f"for (int j = lane; j < {spec.cols}; j += {lanes}) {{", red)
    body = em.emit(store_guard="lane == 0")
    L = [f"extern \"C\" __global__ void __launch_bounds__({threads}) cinn_k_row({_params(spec)}) {{"]
    if warp:
        L.append("  const int lane = threadIdx.x & 31;")
        L.append(f"  for (long long row = blockIdx.x * {rpb}LL + (threadIdx.x >> 5); row < rows; row += gridDim.x * {rpb}LL) {{")
    else:
        L.append("  __shared__ double cinn_smem[32];")
        L.append("  const int lane = threadIdx.x;")
        L.append("  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {")
    L.append(body)
    L.append("  }\n}")
    return "\n".join(L), threads, rpb


def _cuda_col_kernels(spec):
    """Column reduction on [A, K, B]: CTAs of 32 columns x 8 k-lanes; `split` CTAs share the K range of one (a, column tile) and leave fp32
    partials that a second, tiny kernel adds up (no atomics: the result is deterministic).  grid = (ceil(B / 32), split, min(A, 65535))."""
    A, K, B = spec.akb
    lines, out_pos = _col_body(spec, "        ")
    parts = ", ".join(f"{compute_type(r.dtype)}* __restrict__ part{r.id}" for r in spec.col)
    L = [f"extern \"C\" __global__ void __launch_bounds__(256) cinn_k_col({_params(spec)}, {parts}, int split) {{", "  (void)rows;"]
    for r in spec.col:
        L.append(f"  __shared__ {compute_type(r.dtype)} sm{r.id}[8][33];")
    L.append("  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;")
    L.append("  const long long b = blockIdx.x * 32LL + tx;")
    L.append(f"  for (long long a = blockIdx.z; a < {A}LL; a += gridDim.z) {{")
    for r in spec.col:
        L.append(f"    {compute_type(r.dtype)} acc{r.id} = 0;")
    L.append(f"    if (b < {B}LL) {{")
    L.append(f"      for (long long k = blockIdx.y * 8LL + ty; k < {K}LL; k += 8LL * split) {{")
    L.append(f"        const long long e = (a * {K}LL + k) * {B}LL + b; const long long row = e / {spec.cols}LL; const long long j = e - row * {spec.cols}LL; (void)row; (void)j;")
    L += lines
    for r in spec.col:
        L.append(f"        acc{r.id} += ({compute_type(r.dtype)})v{r.args[0].id};")
    L.append("      }\n    }")
    for r in spec.col:
        L.append(f"    sm{r.id}[ty][tx] = acc{r.id};")
    L.append("    __syncthreads();")
    L.append(f"    if (ty == 0 && b < {B}LL) {{")
    for r in spec.col:
        T = compute_type(r.dtype)
        L.append(f"      {T} s{r.id} = 0;\n#pragma unroll\n      for (int t = 0; t < 8; ++t) s{r.id} += sm{r.id}[t][tx];")
        L.append(f"      part{r.id}[((long long)blockIdx.y * {A}LL + a) * {B}LL + b] = s{r.id};")
    L.append("    }\n    __syncthreads();\n  }\n}")
    outs = ", ".join(f"{_STORE[r.dtype]}* __restrict__ out{out_pos[r.id]}, const {compute_type(r.dtype)}* __restrict__ part{r.id}" for r in spec.col)
    L.append(f"extern \"C\" __global__ void __launch_bounds__(256) cinn_k_colfin({outs}, int split) {{")
    L.append(f"  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < {A * B}LL; i += gridDim.x * 256LL) {{")
    for r in spec.col:
        T = compute_type(r.dtype)
        sc = r.attrs.get("scale")
        L.append(f"    {T} s{r.id} = 0; for (int p = 0; p < split; ++p) s{r.id} += part{r.id}[(long long)p * {A * B}LL + i];")
        L.append(f"    st(out{out_pos[r.id]}, i, s{r.id}{'' if sc is None else ' * ' + _lit(sc, T)});")
    L.append("  }\n}")
    n_out = len(spec.outputs)
    part_args = ", ".join(f"({compute_type(r.dtype)}*)out[{n_out + i}]" for i, r in enumerate(spec.col))
    fin_args = ", ".join(f"({_STORE[r.dtype]}*)out[{out_pos[r.id]}], (const {compute_type(r.dtype)}*)out[{n_out + i}]" for i, r in enumerate(spec.col))
    launch = (f"  const int split = aux < 1 ? 1 : aux;\n"
              f"  dim3 grid((unsigned)(({B}LL + 31) / 32), (unsigned)split, (unsigned)({min(A, 65535)}));\n"
              f"  cinn_k_col<<<grid, 256, 0, (cudaStream_t)stream>>>({_call_args(spec)}, {part_args}, split);\n"
              f"  cinn_k_colfin<<<cinn_grid(({A * B}LL + 255) / 256, {SM_COUNT * 8}), 256, 0, (cudaStream_t)stream>>>({fin_args}, split);\n")
    return "\n".join(L), launch


def col_split(spec, sm_count=SM_COUNT):
    """How many CTAs share the K range of one column tile (launch argument `aux`): enough CTAs to cover the machine twice, at least 16 k per CTA."""
    A, K, B = spec.akb
    tiles = ((B + 31) // 32) * min(A, 65535)
    want = -(-2 * sm_count // max(tiles, 1))
    return int(max(1, min(want, max(1, K // 16), 64)))


def cuda_source(spec):
    """Kernels + an `extern "C"` launcher: cinn_launch(in, out, stream, allow_vec, rows) -> cudaError_t of the launch.  The number of rows
    (product of the leading extents) is a run-time argument and the kernel names are fixed, so groups that differ only in batch / sequence
    extents generate the same source and share one compiled object."""
    cap = SM_COUNT * 8
    clamp = "static inline int cinn_grid(long long want, long long cap) { return (int)(want < 1 ? 1 : (want > cap ? cap : want)); }\n"
    if spec.col:
        k, launch = _cuda_col_kernels(spec)
    elif spec.has_reduce:
        k, threads, rpb = _row_kernel(spec)
        launch = (f"  const int grid = cinn_grid((rows + {rpb - 1}) / {rpb}, {cap * (1 if rpb > 1 else 2)});\n"
                  f"  cinn_k_row<<<grid, {threads}, 0, (cudaStream_t)stream>>>({_call_args(spec)});\n")
    else:
        k = _flat_kernels(spec)
        launch = f"  const long long n = rows * {spec.cols}LL;\n"
        V = _vec_width(spec)
        if V:
            launch += (f"  if (allow_vec) {{ cinn_k_vec{V}<<<cinn_grid((n / {V} + 255) / 256, {cap}), 256, 0, (cudaStream_t)stream>>>({_call_args(spec)}); "
                       "return (int)cudaGetLastError(); }\n")
        launch += f"  cinn_k_flat<<<cinn_grid((n + 255) / 256, {cap}), 256, 0, (cudaStream_t)stream>>>({_call_args(spec)});\n"
    return (_CUDA_PRELUDE + "\n" + k + "\n\n" + clamp + "extern \"C\" int cinn_launch(void** in, void** out, void* stream, int allow_vec, long long rows, int aux) {\n  (void)allow_vec; (void)aux;\n"
            + launch + "  return (int)cudaGetLastError();\n}\n")
