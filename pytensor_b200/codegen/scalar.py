"""Scalar program IR and its translation to CUDA device code.

A `ScalarProgram` is the backend's own, plain-data restatement of the straight-line scalar graph the reference keeps
in `Composite.fgraph` (pytensor/scalar/basic.py:4010-4170) or of a single `ScalarOp`.  The lowering
(pytensor_b200/link/cuda/lower.py) builds it; nothing in this module imports pytensor.

Semantics follow the per-op C expressions the reference's C linker compiles (SURVEY.md appendix C restates them from
`ScalarOp.c_code` in pytensor/scalar/basic.py:1411-3861 and pytensor/scalar/math.py): fp32 graphs use fp32 libm
(`expf`, `tanhf` … through CUDA's overloaded math functions — never fast-math intrinsics), `Maximum`/`Minimum`
propagate NaN, `IntDiv`/`Mod` have Python floor semantics, integer true division goes through double, `Softplus` /
`Log1mexp` use the reference's branch thresholds (scalar/math.py:1253-1282, :1326).
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

CTYPE = {
    "bool": "unsigned char", "int8": "signed char", "int16": "short", "int32": "int", "int64": "long long",
    "uint8": "unsigned char", "uint16": "unsigned short", "uint32": "unsigned int", "uint64": "unsigned long long",
    "float32": "float", "float64": "double",
}
ITEMSIZE = {"bool": 1, "int8": 1, "int16": 2, "int32": 4, "int64": 8, "uint8": 1, "uint16": 2, "uint32": 4,
            "uint64": 8, "float32": 4, "float64": 8, "float16": 2}


def is_float(dt: str) -> bool:
    return dt in ("float32", "float64")


def is_int(dt: str) -> bool:
    return dt.startswith("int") or dt.startswith("uint")


def is_uint(dt: str) -> bool:
    return dt.startswith("uint")


class UnsupportedScalarOp(NotImplementedError):
    pass


@dataclass
class ScalarInst:
    op: str  # reference ScalarOp class name, e.g. "Add", "Tanh", "Cast"
    args: list  # refs: ("i", k) input, ("c", k) constant, ("t", k) temp
    in_dtypes: list
    out_dtype: str


@dataclass
class ScalarProgram:
    in_dtypes: list
    out_dtypes: list
    consts: list = field(default_factory=list)  # (dtype, python value)
    insts: list = field(default_factory=list)  # ScalarInst; result of inst k is ("t", k)
    outputs: list = field(default_factory=list)  # refs

    def signature(self) -> str:
        return repr((self.in_dtypes, self.out_dtypes, [(d, repr(v)) for d, v in self.consts],
                     [(i.op, i.args, i.in_dtypes, i.out_dtype) for i in self.insts], self.outputs))

    def n_transcendental(self) -> int:
        heavy = {"Exp", "Exp2", "Expm1", "Log", "Log2", "Log10", "Log1p", "Tanh", "Sinh", "Cosh", "Sin", "Cos", "Tan",
                 "Pow", "Sigmoid", "Softplus", "Log1mexp", "Erf", "Erfc", "Erfcx", "Erfinv", "Erfcinv", "Gamma",
                 "GammaLn", "ArcSin", "ArcCos", "ArcTan", "ArcTan2", "ArcSinh", "ArcCosh", "ArcTanh", "J0", "J1",
                 "I0", "I1", "Psi", "TriGamma", "GammaInc", "GammaIncC", "BetaInc", "Sqrt", "TrueDiv", "Reciprocal"}
        return sum(1 for i in self.insts if i.op in heavy)


# ---- literals -------------------------------------------------------------------------------------------------------
def literal(dtype: str, value) -> str:
    if dtype == "bool":
        return "((unsigned char)1)" if bool(value) else "((unsigned char)0)"
    if is_int(dtype):
        v = int(value)
        ct = CTYPE[dtype]
        if dtype == "uint64":
            return f"(({ct}){v}ULL)"
        if dtype == "int64":
            if v == -(2 ** 63):
                return "((long long)(-9223372036854775807LL - 1LL))"
            return f"(({ct}){v}LL)"
        return f"(({ct}){v})"
    v = float(value)
    if dtype == "float32":
        if math.isnan(v):
            return "__int_as_float(0x7fc00000)"
        if math.isinf(v):
            return "__int_as_float(0x7f800000)" if v > 0 else "__int_as_float(0xff800000)"
        return f"{np.float32(v).item().hex()}f" if v != 0 else ("-0.0f" if math.copysign(1.0, v) < 0 else "0.0f")
    if dtype == "float64":
        if math.isnan(v):
            return "__longlong_as_double(0x7ff8000000000000LL)"
        if math.isinf(v):
            return "__longlong_as_double(0x7ff0000000000000LL)" if v > 0 else "__longlong_as_double(0xfff0000000000000LL)"
        return f"{v.hex()}" if v != 0 else ("-0.0" if math.copysign(1.0, v) < 0 else "0.0")
    raise UnsupportedScalarOp(f"constant of dtype {dtype}")


# ---- per-op expression table -----------------------------------------------------------------------------------------
def _nan(dt):
    return "__int_as_float(0x7fc00000)" if dt == "float32" else "__longlong_as_double(0x7ff8000000000000LL)"


def _unary_libm(fn):
    def emit(a, it, ot):
        T = CTYPE[ot]
        return f"{fn}(({T})({a[0]}))"
    return emit


def _cmp(sym):
    def emit(a, it, ot):
        return f"((unsigned char)(({a[0]}) {sym} ({a[1]})))"
    return emit


def _add(a, it, ot):
    if ot == "bool":
        return "((unsigned char)(" + " || ".join(f"({x})" for x in a) + "))"
    return "(" + " + ".join(f"({x})" for x in a) + ")"


def _mul(a, it, ot):
    if ot == "bool":
        return "((unsigned char)(" + " && ".join(f"({x})" for x in a) + "))"
    return "(" + " * ".join(f"({x})" for x in a) + ")"


def _truediv(a, it, ot):
    if all(not is_float(t) for t in it):
        return f"(((double)({a[0]})) / ({a[1]}))"
    return f"(({a[0]}) / ({a[1]}))"


def _intdiv(a, it, ot):
    x, y = a
    if is_float(ot):
        if not any(is_float(t) for t in it):
            # two INTEGER operands whose common type is a float (int64 with uint64): the quotient is C's integer division,
            # like in the reference's `floor(x / y)`; the explicit double keeps floor() unambiguous for the device compiler
            return f"floor((double)(({x}) / ({y})))"
        return f"floor(({x}) / ({y}))"
    if ot == "bool" or is_uint(ot):
        return f"(({y}) == 0 ? 0 : ({x}) / ({y}))"
    T = CTYPE[ot]
    return (f"ptk_floordiv<{T}>(({T})({x}), ({T})({y}))")


def _mod(a, it, ot):
    x, y = a
    T = CTYPE[ot]
    if is_float(ot):
        return f"ptk_fmod_py<{T}>(({T})({x}), ({T})({y}))"
    if ot == "bool" or is_uint(ot):
        return f"(({y}) == 0 ? 0 : ({x}) % ({y}))"
    return f"ptk_imod_py<{T}>(({T})({x}), ({T})({y}))"


def _mixed_signedness(it) -> bool:
    return any(is_uint(t) for t in it) and any(is_int(t) and not is_uint(t) for t in it)


def _maximum(a, it, ot):
    x, y = a
    if ot == "float32" and all(t == "float32" for t in it):
        return f"ptk_max_nan_f32(({x}), ({y}))"  # one FMNMX.NAN: NaN-propagating like the reference's Maximum.c_code
    if is_float(ot):
        return f"((({y}) > ({x})) ? ({y}) : ((({x}) >= ({y})) ? ({x}) : {_nan(ot)}))"
    if _mixed_signedness(it):
        # the reference's expression VERBATIM in meaning (scalar/basic.py Maximum.c_code: one expression with a nan("")
        # arm for every dtype): the comparison happens in the unsigned type, but the selected operand reaches the integer
        # result through the double the nan arm forces — so a negative signed operand keeps its sign
        return f"((({y}) > ({x})) ? (double)({y}) : ((({x}) >= ({y})) ? (double)({x}) : {_nan('float64')}))"
    return f"((({y}) > ({x})) ? ({y}) : ({x}))"


def _minimum(a, it, ot):
    x, y = a
    if ot == "float32" and all(t == "float32" for t in it):
        return f"ptk_min_nan_f32(({x}), ({y}))"
    if is_float(ot):
        return f"((({y}) < ({x})) ? ({y}) : ((({x}) <= ({y})) ? ({x}) : {_nan(ot)}))"
    if _mixed_signedness(it):   # (see _maximum)
        return f"((({y}) < ({x})) ? (double)({y}) : ((({x}) <= ({y})) ? (double)({x}) : {_nan('float64')}))"
    return f"((({y}) < ({x})) ? ({y}) : ({x}))"


def _abs(a, it, ot):
    if is_float(it[0]):
        return f"fabs({a[0]})"
    if it[0] == "bool" or is_uint(it[0]):
        return f"({a[0]})"
    return f"((({a[0]}) < 0) ? -({a[0]}) : ({a[0]}))"


def _sign(a, it, ot):
    x = a[0]
    if is_float(it[0]):
        T = CTYPE[ot]
        return f"((({x}) > 0) ? ({T})1 : ((({x}) < 0) ? ({T})-1 : (isnan({x}) ? {_nan(ot)} : ({T})0)))"
    if it[0] == "bool" or is_uint(it[0]):
        return f"((({x}) > 0) ? 1 : 0)"
    return f"((({x}) > 0) - (({x}) < 0))"


def _cast(a, it, ot):
    if ot == "bool":
        return f"((unsigned char)(({a[0]}) ? 1 : 0))"
    return f"(({CTYPE[ot]})({a[0]}))"


def _isnan(a, it, ot):
    if is_float(it[0]):
        return f"((unsigned char)(isnan({a[0]}) ? 1 : 0))"
    return "((unsigned char)0)"


def _isinf(a, it, ot):
    if is_float(it[0]):
        return f"((unsigned char)(isinf({a[0]}) ? 1 : 0))"
    return "((unsigned char)0)"


def _invert(a, it, ot):
    if it[0] == "bool":
        return f"((unsigned char)(!({a[0]})))"
    return f"(~({a[0]}))"


def _trunc(a, it, ot):
    return f"trunc({a[0]})"


def _sigmoid(a, it, ot):
    T = CTYPE[ot]
    return f"(({T})1 / (({T})1 + exp(-(({T})({a[0]})))))"


def _softplus(a, it, ot):
    T = CTYPE[ot]
    x = f"(({T})({a[0]}))"
    s = "f" if ot == "float32" else ""
    return (f"(({x} < -37.0{s}) ? exp({x}) : (({x} < 18.0{s}) ? log1p(exp({x})) : "
            f"(({x} < 33.3{s}) ? ({x} + exp(-{x})) : {x})))")


def _log1mexp(a, it, ot):
    T = CTYPE[ot]
    x = f"(({T})({a[0]}))"
    s = "f" if ot == "float32" else ""
    return f"(({x} < -0.6931471805599453{s}) ? log1p(-exp({x})) : log(-expm1({x})))"


def _pow(a, it, ot):
    T = CTYPE[ot]
    if is_float(ot):
        return f"pow(({T})({a[0]}), ({T})({a[1]}))"
    return f"(({T})pow((double)({a[0]}), (double)({a[1]})))"


def _recip(a, it, ot):
    T = CTYPE[ot]
    return f"(({T})1 / ({T})({a[0]}))"


def _round_even(a, it, ot):
    return f"rint({a[0]})"


OPS = {
    "Add": _add, "Mul": _mul,
    "Sub": lambda a, it, ot: f"(({a[0]}) - ({a[1]}))",
    "Neg": lambda a, it, ot: f"(-({a[0]}))",
    "Sqr": lambda a, it, ot: f"(({a[0]}) * ({a[0]}))",
    "Reciprocal": _recip, "TrueDiv": _truediv, "IntDiv": _intdiv, "Mod": _mod, "Pow": _pow,
    "Identity": lambda a, it, ot: f"({a[0]})",
    "Conj": lambda a, it, ot: f"({a[0]})",
    "Second": lambda a, it, ot: f"({a[1]})",
    "Abs": _abs, "Sign": _sign, "Cast": _cast,
    "LT": _cmp("<"), "GT": _cmp(">"), "LE": _cmp("<="), "GE": _cmp(">="), "EQ": _cmp("=="), "NEQ": _cmp("!="),
    "IsNan": _isnan, "IsInf": _isinf,
    "AND": lambda a, it, ot: f"(({a[0]}) & ({a[1]}))",
    "OR": lambda a, it, ot: f"(({a[0]}) | ({a[1]}))",
    "XOR": lambda a, it, ot: f"(({a[0]}) ^ ({a[1]}))",
    "Invert": _invert,
    "Switch": lambda a, it, ot: f"(({a[0]}) ? ({a[1]}) : ({a[2]}))",
    "Clip": lambda a, it, ot: f"((({a[0]}) < ({a[1]})) ? ({a[1]}) : ((({a[0]}) > ({a[2]})) ? ({a[2]}) : ({a[0]})))",
    "Maximum": _maximum, "Minimum": _minimum,
    "Ceil": _unary_libm("ceil"), "Floor": _unary_libm("floor"), "Trunc": _trunc,
    "RoundHalfAwayFromZero": _unary_libm("round"), "RoundHalfToEven": _round_even,
    "Exp": _unary_libm("exp"), "Exp2": _unary_libm("exp2"), "Expm1": _unary_libm("expm1"),
    "Log": _unary_libm("log"), "Log2": _unary_libm("log2"), "Log10": _unary_libm("log10"),
    "Log1p": _unary_libm("log1p"), "Sqrt": _unary_libm("sqrt"),
    "Sin": _unary_libm("sin"), "Cos": _unary_libm("cos"), "Tan": _unary_libm("tan"),
    "ArcSin": _unary_libm("asin"), "ArcCos": _unary_libm("acos"), "ArcTan": _unary_libm("atan"),
    "ArcTan2": lambda a, it, ot: f"atan2(({CTYPE[ot]})({a[0]}), ({CTYPE[ot]})({a[1]}))",
    "Sinh": _unary_libm("sinh"), "Cosh": _unary_libm("cosh"), "Tanh": _unary_libm("tanh"),
    "ArcSinh": _unary_libm("asinh"), "ArcCosh": _unary_libm("acosh"), "ArcTanh": _unary_libm("atanh"),
    "Sigmoid": _sigmoid, "Softplus": _softplus, "Log1mexp": _log1mexp,
    "Erf": _unary_libm("erf"), "Erfc": _unary_libm("erfc"), "Erfcx": _unary_libm("erfcx"),
    "Erfinv": _unary_libm("erfinv"), "Erfcinv": _unary_libm("erfcinv"),
    "Gamma": _unary_libm("tgamma"), "GammaLn": _unary_libm("lgamma"),
    "J0": _unary_libm("j0"), "J1": _unary_libm("j1"),
    "I0": _unary_libm("cyl_bessel_i0"), "I1": _unary_libm("cyl_bessel_i1"),
    # special functions the reference computes in DOUBLE whatever the graph dtype (scalar/math.py:490 `_psi`, :574
    # `_tri_gamma`, :648 `GammaP`, :695 `GammaQ`, :1371 `BetaInc`) — device versions in SPECIAL_HELPERS below
    "Psi": lambda a, it, ot: f"ptk_psi((double)({a[0]}))",
    "TriGamma": lambda a, it, ot: f"ptk_trigamma((double)({a[0]}))",
    "GammaInc": lambda a, it, ot: f"ptk_gamma_p((double)({a[0]}), (double)({a[1]}))",
    "GammaIncC": lambda a, it, ot: f"ptk_gamma_q((double)({a[0]}), (double)({a[1]}))",
    "BetaInc": lambda a, it, ot: f"ptk_betainc((double)({a[0]}), (double)({a[1]}), (double)({a[2]}))",
}

# which helper blocks (SPECIAL_HELPERS) an op's expression needs
NEEDS = {"Psi": ("psi",), "TriGamma": ("trigamma",), "GammaInc": ("gammainc",), "GammaIncC": ("gammainc",),
         "BetaInc": ("betainc",)}


# Device restatements of the reference's double-precision special functions.  Emitted in front of a scalar body only when
# the body uses them (they are fp64-heavy; keeping them out of every other kernel keeps NVRTC time and register use down).
SPECIAL_HELPERS = {
    # Psi: Bernardo's AS 103 exactly as the reference evaluates it (scalar/math.py:441-487): truncated Stirling
    # coefficients, recurrence up to 8.5, +inf at non-positive integers, reflection psi(x) = psi(1-x) - pi*cot(pi*x).
    "psi": r"""
#ifndef PTK_HAVE_PSI
#define PTK_HAVE_PSI
__device__ inline double ptk_psi(double x) {
  double acc = 0.0;
  if (x <= 0.0) {
    if (x == floor(x)) return __longlong_as_double(0x7ff0000000000000LL);
    const double px = 3.14159265358979323846 * x;
    acc = -3.14159265358979323846 * (cos(px) / sin(px));
    x = 1.0 - x;
  }
  if (x <= 1.0e-5) return (-0.5772156649 - 1.0 / x) + acc;
  double s = 0.0;
  while (x < 8.5) { s -= 1.0 / x; x += 1.0; }
  const double r = 1.0 / x, r2 = r * r;
  s = s + log(x) - 0.5 * r;
  s = s - r2 * (8.333333333e-2 - r2 * (8.333333333e-3 - r2 * 3.968253968e-3));
  return s + acc;
}
#endif
""",
    # TriGamma: AS 121 as in scalar/math.py:529-566 (0 for x <= 0, 1/x^2 below 1e-4, recurrence up to 5, 4-term asymptote)
    "trigamma": r"""
#ifndef PTK_HAVE_TRIGAMMA
#define PTK_HAVE_TRIGAMMA
__device__ inline double ptk_trigamma(double x) {
  if (x <= 0.0) return 0.0;
  if (x <= 0.0001) return 1.0 / x / x;
  double v = 0.0;
  while (x < 5.0) { v += 1.0 / x / x; x += 1.0; }
  const double y = 1.0 / x / x;
  return v + (0.5 * y + (1.0 + y * (0.1666666667 + y * (-0.03333333333 + y * (0.02380952381 + y * -0.03333333333)))) / x);
}
#endif
""",
    # Regularised incomplete gamma P / Q (scalar/c_code/gamma.c:228-254): series for x < a+1, modified-Lentz continued
    # fraction otherwise, same argument checks and limits; ln Gamma(a) from CUDA's lgamma instead of the table+Lanczos
    # of gamma.c:83-104 (both are accurate far beyond the 1e-5 bar).
    "gammainc": r"""
#ifndef PTK_HAVE_GAMMAINC
#define PTK_HAVE_GAMMAINC
__device__ inline double ptk_gamma_series(double a, double x) {
  double term = 1.0 / a, sum = term;
  for (int i = 0; i < 1024; ++i) {
    a += 1.0;
    term *= x / a;
    sum += term;
    if (fabs(term) < fabs(sum) * 2.2204460492503131e-16) break;
  }
  return sum;
}
__device__ inline double ptk_gamma_cfrac(double a, double x) {
  const double tiny = 2.2204460492503131e-16 * 2.2204460492503131e-16 * 2.2204460492503131e-16;
  double b = x + 1.0 - a, c = 1.0 / tiny, d = 1.0 / b, f = d;
  for (int i = 1; i < 1024; ++i) {
    const double an = i * (a - i);
    b += 2.0;
    d = an * d + b;
    if (fabs(d) < tiny) d = tiny;
    c = b + an / c;
    if (fabs(c) < tiny) c = tiny;
    d = 1.0 / d;
    const double e = d * c;
    f *= e;
    if (fabs(e - 1.0) < 2.2204460492503131e-16) break;
  }
  return f;
}
// which = 0: P (lower), 1: Q (upper)
__device__ inline double ptk_gamma_pq(double a, double x, int which) {
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  if (a <= 0.0 || x < 0.0) return nan;
  if (x <= 0.0) return which ? 1.0 : 0.0;
  if (isinf(a)) return isinf(x) ? nan : (which ? 1.0 : 0.0);
  if (isinf(x)) return which ? 0.0 : 1.0;
  const double pref = exp(a * log(x) - x - lgamma(a));
  if (x < a + 1.0) {
    const double p = ptk_gamma_series(a, x) * pref;
    return which ? 1.0 - p : p;
  }
  const double q = ptk_gamma_cfrac(a, x) * pref;
  return which ? q : 1.0 - q;
}
__device__ inline double ptk_gamma_p(double a, double x) { return ptk_gamma_pq(a, x, 0); }
__device__ inline double ptk_gamma_q(double a, double x) { return ptk_gamma_pq(a, x, 1); }
#endif
""",
    # Regularised incomplete beta (scalar/c_code/incbet.c:34-93, Cephes `incbet`): power series when b*x <= 1 and
    # x <= 0.95; otherwise reflect about the mean, pick one of the two continued fractions by the sign of
    # x(a+b-2)-(a-1), and scale by x^a (1-x)^b / (a B(a,b)) directly or through logarithms when that would overflow.
    "betainc": r"""
#ifndef PTK_HAVE_BETAINC
#define PTK_HAVE_BETAINC
__device__ inline double ptk_betainc_pseries(double a, double b, double x) {
  const double ai = 1.0 / a, eps = 1.11022302462515654042e-16;
  double u = (1.0 - b) * x, t = u, v = u / (a + 1.0), n = 2.0, s = 0.0;
  const double first = v, stop = eps * ai;
  while (fabs(v) > stop) {
    t *= (n - b) * x / n;
    v = t / (a + n);
    s += v;
    n += 1.0;
  }
  s += first;
  s += ai;
  const double lx = a * log(x);
  if (a + b < 171.624376956302725 && fabs(lx) < 7.09782712893383996732e2)
    return s * (tgamma(a + b) / (tgamma(a) * tgamma(b))) * pow(x, a);
  const double lt = lgamma(a + b) - lgamma(a) - lgamma(b) + lx + log(s);
  return lt < -7.451332191019412076235e2 ? 0.0 : exp(lt);
}
// Forward evaluation of a continued fraction 1/(1+ d1/(1+ d2/(1+ ...))) whose partial numerators come in (odd, even)
// pairs; `second` selects the expansion in z = x/(1-x).  Numerators and denominators are rescaled by 2^+-52 when they
// leave [2^-52, 2^52], as Cephes does, so that neither over- nor underflows.
__device__ inline double ptk_betainc_cf(double a, double b, double x, int second) {
  const double big = 4.503599627370496e15, biginv = 2.22044604925031308085e-16, thresh = 3.0 * 1.11022302462515654042e-16;
  const double z = second ? x / (1.0 - x) : x;
  double k1 = a, k2 = second ? b - 1.0 : a + b, k3 = a, k4 = a + 1.0;
  double k5 = 1.0, k6 = second ? a + b : b - 1.0, k7 = a + 1.0, k8 = a + 2.0;
  const double s2 = second ? -1.0 : 1.0, s6 = second ? 1.0 : -1.0;
  double pm2 = 0.0, qm2 = 1.0, pm1 = 1.0, qm1 = 1.0, ans = 1.0, r = 1.0;
  for (int n = 0; n < 300; ++n) {
    double d = -(z * k1 * k2) / (k3 * k4);
    double pk = pm1 + pm2 * d, qk = qm1 + qm2 * d;
    pm2 = pm1; pm1 = pk; qm2 = qm1; qm1 = qk;
    d = (z * k5 * k6) / (k7 * k8);
    pk = pm1 + pm2 * d; qk = qm1 + qm2 * d;
    pm2 = pm1; pm1 = pk; qm2 = qm1; qm1 = qk;
    if (qk != 0.0) r = pk / qk;
    double t = 1.0;
    if (r != 0.0) { t = fabs((ans - r) / r); ans = r; }
    if (t < thresh) break;
    k1 += 1.0; k2 += s2; k3 += 2.0; k4 += 2.0; k5 += 1.0; k6 += s6; k7 += 2.0; k8 += 2.0;
    if (fabs(qk) + fabs(pk) > big) { pm2 *= biginv; pm1 *= biginv; qm2 *= biginv; qm1 *= biginv; }
    if (fabs(qk) < biginv || fabs(pk) < biginv) { pm2 *= big; pm1 *= big; qm2 *= big; qm1 *= big; }
  }
  return ans;
}
__device__ inline double ptk_betainc(double a, double b, double x) {
  const double nan = __longlong_as_double(0x7ff8000000000000LL), eps = 1.11022302462515654042e-16;
  if (a <= 0.0 || b <= 0.0 || x < 0.0 || 1.0 < x) return nan;
  if (x == 0.0) return 0.0;
  if (x == 1.0) return 1.0;
  if (b * x <= 1.0 && x <= 0.95) return ptk_betainc_pseries(a, b, x);
  // at most one reflection: after swapping, x' = 1-x <= b/(a+b) = the new mean, so the second pass never reflects
  bool flipped = false;
  double xc = 1.0 - x;
  if (x > a / (a + b)) {
    flipped = true;
    const double t0 = a; a = b; b = t0;
    const double t1 = x; x = xc; xc = t1;
    if (b * x <= 1.0 && x <= 0.95) {
      const double t = ptk_betainc_pseries(a, b, x);
      return t <= eps ? 1.0 - eps : 1.0 - t;
    }
  }
  const double w = (x * (a + b - 2.0) - (a - 1.0) < 0.0) ? ptk_betainc_cf(a, b, x, 0) : ptk_betainc_cf(a, b, x, 1) / xc;
  double y = a * log(x), t = b * log(xc);
  if (a + b < 171.624376956302725 && fabs(y) < 7.09782712893383996732e2 && fabs(t) < 7.09782712893383996732e2) {
    t = pow(xc, b);
    t *= pow(x, a);
    t /= a;
    t *= w;
    t *= tgamma(a + b) / (tgamma(a) * tgamma(b));
  } else {
    y += t + lgamma(a + b) - lgamma(a) - lgamma(b);
    y += log(w / a);
    t = y < -7.451332191019412076235e2 ? 0.0 : exp(y);
  }
  if (flipped) return t <= eps ? 1.0 - eps : 1.0 - t;
  return t;
}
#endif
""",
}

PRELUDE = r"""
// ---- ptk scalar helpers ----
__device__ __forceinline__ float ptk_max_nan_f32(float a, float b) { float r; asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float ptk_min_nan_f32(float a, float b) { float r; asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
// Python floor-division / modulo semantics of IntDiv / Mod
template <typename T> __device__ __forceinline__ T ptk_floordiv(T x, T y) {
  if (y == 0) return 0;
  T q = x / y;
  if ((x % y != 0) && ((x < 0) != (y < 0))) --q;
  return q;
}
template <typename T> __device__ __forceinline__ T ptk_imod_py(T x, T y) {
  if (y == 0) return 0;
  T r = x % y;
  if (r != 0 && ((r < 0) != (y < 0))) r += y;
  return r;
}
template <typename T> __device__ __forceinline__ T ptk_fmod_py(T x, T y) {
  if (y == 0) return x - x + (T)__int_as_float(0x7fc00000);
  T r = fmod(x, y);
  if (r != 0 && ((r < 0) != (y < 0))) r += y;
  return r;
}
"""


def _ref_expr(ref, prog: ScalarProgram) -> str:
    kind, k = ref
    if kind == "i":
        return f"i{k}"
    if kind == "c":
        d, v = prog.consts[k]
        return literal(d, v)
    return f"t{k}"


def emit_body(prog: ScalarProgram, fn_name: str = "ptk_body") -> str:
    """`__device__ void fn(const T0& i0, ..., O0& o0, ...)` computing all outputs of `prog`."""
    for d in list(prog.in_dtypes) + list(prog.out_dtypes) + [i.out_dtype for i in prog.insts]:
        if d not in CTYPE:
            raise UnsupportedScalarOp(f"dtype {d} has no device path (the reference's C linker has none for float16/complex either)")
    params = [f"const {CTYPE[d]} i{k}" for k, d in enumerate(prog.in_dtypes)]
    params += [f"{CTYPE[d]}& o{k}" for k, d in enumerate(prog.out_dtypes)]
    need = []
    for inst in prog.insts:
        for h in NEEDS.get(inst.op, ()):
            if h not in need:
                need.append(h)
    lines = [SPECIAL_HELPERS[h] for h in need]
    lines.append(f"__device__ __forceinline__ void {fn_name}({', '.join(params)}) {{")
    for k, inst in enumerate(prog.insts):
        fn = OPS.get(inst.op)
        if fn is None:
            raise UnsupportedScalarOp(f"scalar op {inst.op} has no sm_90a device expression yet")
        args = [_ref_expr(r, prog) for r in inst.args]
        expr = fn(args, inst.in_dtypes, inst.out_dtype)
        T = CTYPE[inst.out_dtype]
        lines.append(f"  const {T} t{k} = ({T})({expr});")
    for k, ref in enumerate(prog.outputs):
        lines.append(f"  o{k} = ({CTYPE[prog.out_dtypes[k]]})({_ref_expr(ref, prog)});")
    lines.append("}")
    return "\n".join(lines)


def simplify(prog: ScalarProgram) -> ScalarProgram:
    """Exact algebraic peepholes over a ScalarProgram (every IEEE operation of the simplified program returns what the
    unsimplified one returns, for EVERY input: NaNs, infinities, denormals), applied once at lowering time:

      Maximum(u, -u) -> Abs(u)     where -u is `Neg(u)`, or u = c * x and -u = (-c) * x with literal constants of the
                                   operands' own floating-point type.  IEEE multiplication is sign-symmetric, so (-c) * x is
                                   exactly -(c * x); max(y, -y) is |y|: NaN for a NaN (the reference's Maximum propagates
                                   NaNs, scalar/basic.py ScalarMaximum.c_code) and +0 for y = +-0, which is also what
                                   the device's max.NaN instruction returns for (-0, +0) in either order.

    The instruction that computed -u stays in the program (its result may have other readers); the device compiler drops
    it when it has none.  PTK_SCALAR_SIMPLIFY=0 disables."""
    import os

    if os.environ.get("PTK_SCALAR_SIMPLIFY", "1") == "0":
        return prog
    insts = prog.insts

    def const_value(ref, dtype):
        if ref[0] != "c":
            return None
        d, v = prog.consts[ref[1]]
        return v if d == dtype and isinstance(v, float) else None

    def mul_parts(ref, dtype):
        """(constant value, other operand ref) of `c * x` / `x * c` computed in `dtype`, else None."""
        if ref[0] != "t":
            return None
        i = insts[ref[1]]
        if i.op != "Mul" or len(i.args) != 2 or i.out_dtype != dtype or list(i.in_dtypes) != [dtype, dtype]:
            return None
        for a, b in ((0, 1), (1, 0)):
            c = const_value(i.args[a], dtype)
            if c is not None and i.args[b][0] != "c":
                return c, tuple(i.args[b])
        return None

    def is_neg_of(a, b, dtype):
        """Is the value of ref a exactly -(value of ref b)?"""
        if a[0] == "t":
            i = insts[a[1]]
            if i.op == "Neg" and i.out_dtype == dtype and list(i.in_dtypes) == [dtype] and tuple(i.args[0]) == tuple(b):
                return True
        pa, pb = mul_parts(a, dtype), mul_parts(b, dtype)
        return pa is not None and pb is not None and pa[1] == pb[1] and pa[0] == -pb[0] and pa[0] == pa[0]

    out = None
    for k, i in enumerate(insts):
        if i.op == "Maximum" and len(i.args) == 2 and i.out_dtype in ("float32", "float64") \
                and list(i.in_dtypes) == [i.out_dtype, i.out_dtype]:
            a, b = tuple(i.args[0]), tuple(i.args[1])
            if is_neg_of(b, a, i.out_dtype) or is_neg_of(a, b, i.out_dtype):
                if out is None:
                    out = list(insts)
                keep = a if a[0] == "t" or b[0] != "t" else b
                out[k] = ScalarInst("Abs", [keep], [i.out_dtype], i.out_dtype)
    if out is None:
        return prog
    return ScalarProgram(list(prog.in_dtypes), list(prog.out_dtypes), list(prog.consts), out, list(prog.outputs))


def single_op_program(op: str, in_dtypes, out_dtype) -> ScalarProgram:
    return ScalarProgram(
        in_dtypes=list(in_dtypes), out_dtypes=[out_dtype],
        insts=[ScalarInst(op, [("i", k) for k in range(len(in_dtypes))], list(in_dtypes), out_dtype)],
        outputs=[("t", 0)],
    )
