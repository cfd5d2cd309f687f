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
    # the reference evaluates these four through SciPy (scalar/math.py PolyGamma, GammaIncInv, GammaIncCInv, BetaIncInv
    # have no C code), in double whatever the graph dtype
    "PolyGamma": lambda a, it, ot: f"ptk_polygamma((long long)({a[0]}), (double)({a[1]}))",
    "GammaIncInv": lambda a, it, ot: f"ptk_gammaincinv((double)({a[0]}), (double)({a[1]}))",
    "GammaIncCInv": lambda a, it, ot: f"ptk_gammainccinv((double)({a[0]}), (double)({a[1]}))",
    "BetaIncInv": lambda a, it, ot: f"ptk_betaincinv((double)({a[0]}), (double)({a[1]}), (double)({a[2]}))",
}

# which helper blocks (SPECIAL_HELPERS) an op's expression needs
NEEDS = {"Psi": ("psi",), "TriGamma": ("trigamma",), "GammaInc": ("gammainc",), "GammaIncC": ("gammainc",),
         "BetaInc": ("betainc",), "PolyGamma": ("polygamma",), "GammaIncInv": ("gammainc", "gammaincinv"),
         "GammaIncCInv": ("gammainc", "gammaincinv"), "BetaIncInv": ("betainc", "betaincinv")}


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
    # PolyGamma(n, x), SciPy's definition: digamma for n = 0, (-1)^(n+1) n! zeta(n+1, x) for n >= 1, NaN for n < 0.
    # Digamma: reflection psi(x) = psi(1-x) - pi cot(pi x) for x < 0 (-inf at +0, +inf at -0, NaN at negative
    # integers), a Taylor series about the positive root x0 = 1.4616... within 0.1 of it (so the result keeps its
    # relative accuracy where it crosses zero), else the recurrence up to 10 and the asymptotic series.
    # Hurwitz zeta: Euler-Maclaurin summation.  Direct terms (q+k)^-s until q+k >= 10+s or they stop contributing, then
    # the integral, half-term and 12 Bernoulli corrections; +inf at non-positive integer q (and -inf), as in SciPy.
    # Trip caps: the direct sum stops after 256 terms (NaN when q + 256 is still below 10+s: non-integer q < -230 for
    # small n), the Bernoulli loop after 12; digamma's recurrence runs at most 10 times.  The product form keeps SciPy's
    # overflow (n! = inf from n = 171) and 0 * inf = NaN (zeta underflowing for large n and x).
    "polygamma": r"""
#ifndef PTK_HAVE_POLYGAMMA
#define PTK_HAVE_POLYGAMMA
__device__ inline double ptk_digamma(double x) {
  const double inf = __longlong_as_double(0x7ff0000000000000LL), pi = 3.14159265358979323846;
  if (isnan(x)) return x;
  if (x == 0.0) return signbit(x) ? inf : -inf;
  double acc = 0.0;
  if (x < 0.0) {
    if (x == floor(x)) return __longlong_as_double(0x7ff8000000000000LL);
    acc = -pi * cospi(x) / sinpi(x);
    x = 1.0 - x;
  }
  const double h = (x - 1.4616321449683622) - 9.549995429965697e-17;
  if (fabs(h) < 0.1) {
    const double c[14] = {0.9676722454476212, -0.4427631689835921, 0.258499760955651, -0.16394270544240652,
                          0.10782405069126237, -0.07219956125645471, 0.04880428816414311, -0.03316112647484736,
                          0.022597648232218104, -0.01542476590494896, 0.010538791616612175, -0.007204534386356869,
                          0.004926781395729853, -0.003369801655439328};
    double s = c[13];
    for (int k = 12; k >= 0; --k) s = s * h + c[k];
    return s * h + acc;
  }
  double s = 0.0;
  for (int k = 0; k < 10 && x < 10.0; ++k) { s -= 1.0 / x; x += 1.0; }
  const double r2 = 1.0 / (x * x);
  const double t = r2 * (0.08333333333333333 + r2 * (-0.008333333333333333 + r2 * (0.003968253968253968 +
                   r2 * (-0.004166666666666667 + r2 * (0.007575757575757576 + r2 * (-0.021092796092796094 +
                   r2 * 0.08333333333333333))))));
  return (s + (log(x) - 0.5 / x - t)) + acc;
}
// zeta(s, q) = sum_{k >= 0} (q + k)^-s for s >= 2
__device__ inline double ptk_hurwitz_zeta(double s, double q) {
  const double eps = 1.1102230246251565e-16;
  if (isnan(q)) return q;
  if (q <= 0.0 && q == floor(q)) return __longlong_as_double(0x7ff0000000000000LL);
  if (isinf(q)) return 0.0;
  const double W = 10.0 + s;
  double sum = 0.0, w = q;
  for (int k = 0; k < 256 && w < W; ++k) {
    const double t = pow(w, -s);
    sum += t;
    w += 1.0;
    if (w > 1.0 && fabs(t) <= eps * fabs(sum)) return sum;
  }
  if (w < W) return __longlong_as_double(0x7ff8000000000000LL);
  const double b2j[12] = {0.08333333333333333, -0.001388888888888889, 3.306878306878307e-05, -8.267195767195768e-07,
                          2.08767569878681e-08, -5.284190138687493e-10, 1.3382536530684679e-11, -3.3896802963225827e-13,
                          8.586062056277845e-15, -2.174868698558062e-16, 5.5090028283602295e-18, -1.3954464685812522e-19};
  const double a = pow(w, -s);
  sum += w * a / (s - 1.0) + 0.5 * a;
  double f = s * a / w;  // (s)_(2j-1) w^(-s-2j+1)
  for (int j = 0; j < 12; ++j) {
    const double t = f * b2j[j];
    sum += t;
    if (fabs(t) <= eps * fabs(sum)) break;
    f *= (s + 2.0 * j + 1.0) * (s + 2.0 * j + 2.0) / (w * w);
  }
  return sum;
}
__device__ inline double ptk_polygamma(long long n, double x) {
  if (n == 0) return ptk_digamma(x);
  if (n < 0) return __longlong_as_double(0x7ff8000000000000LL);
  const double s = (double)n + 1.0;
  return ((n & 1) ? 1.0 : -1.0) * tgamma(s) * ptk_hurwitz_zeta(s, x);
}
#endif
""",
    # Inverse regularised incomplete gamma (needs "gammainc").  One solver for both tails: it targets whichever of P and
    # Q = 1 - P is <= 1/2 at the solution (1 - t is exact there), so neither tail loses digits to the other.  Unknown
    # u = log x; residual g(u) = +-(log T(e^u) - log t), where log T is formed here as the log prefactor
    # a u - x - lgamma(a) plus the log of ptk_gamma_series / ptk_gamma_cfrac, so far tails do not underflow.  Start
    # (after DiDonato & Morris 1986, Temme 1992): (P Gamma(a+1))^(1/a) for small x; Wilson-Hilferty with the
    # Abramowitz-Stegun 26.2.23 normal deviate for a > 1; the log-tail form x = -log(Q Gamma(a)) + (a-1) log x for
    # the upper tail of a <= 1.  Then Halley steps in u, kept inside a bracket [lo, hi] that every evaluation narrows
    # (a step that leaves it bisects), over u in [-745.2, 709.8].  At most 64 iterations: worst case 64 evaluations of
    # the series or continued fraction (each capped at 1024 terms) per element.
    "gammaincinv": r"""
#ifndef PTK_HAVE_GAMMAINCINV
#define PTK_HAVE_GAMMAINCINV
// log P (which = 0) or log Q (which = 1) at x, given the log prefactor lpref = a log x - x - lgamma(a); *e gets
// |d log T / d log x| = exp(lpref - log T), taken from the series or fraction itself where log T is lpref plus its log
// (the difference of the two logs would cancel for large x)
__device__ inline double ptk_gamma_logpq(double a, double x, double lpref, int which, double* e) {
  if (x < a + 1.0) {
    const double s = ptk_gamma_series(a, x), lp = lpref + log(s);
    if (!which) { *e = 1.0 / s; return lp; }
    const double lq = log1p(-exp(lp));
    *e = exp(lpref - lq);
    return lq;
  }
  const double f = ptk_gamma_cfrac(a, x), lq = lpref + log(f);
  if (which) { *e = 1.0 / f; return lq; }
  const double lp = log1p(-exp(lq));
  *e = exp(lpref - lp);
  return lp;
}
// Abramowitz & Stegun 26.2.23: the z > 0 with upper-tail probability t (0 < t <= 1/2), to about 4.5e-4 (a start only)
__device__ inline double ptk_normal_deviate_start(double t) {
  const double r = sqrt(-2.0 * log(t));
  return r - (2.515517 + r * (0.802853 + r * 0.010328)) / (1.0 + r * (1.432788 + r * (0.189269 + r * 0.001308)));
}
// x with P(a, x) = t (which = 0) or Q(a, x) = t (which = 1); a finite and > 0, 0 < t < 1
__device__ inline double ptk_gammaincinv_tail(double a, double t, int which) {
  if (t > 0.5) { t = 1.0 - t; which ^= 1; }
  const double lt = log(t), lga = lgamma(a), sg = which ? -1.0 : 1.0;
  const double us = ((which ? log1p(-t) : lt) + lgamma(a + 1.0)) / a;  // P ~ x^a / Gamma(a+1) for small x
  if (us < -745.2) return 0.0;                                          // below the smallest denormal
  double u = us;
  if (a > 1.0) {
    const double z = which ? ptk_normal_deviate_start(t) : -ptk_normal_deviate_start(t);
    const double c = 1.0 / (9.0 * a), w = 1.0 - c + z * sqrt(c);
    if (w > 0.05) u = log(a) + 3.0 * log(w);
  } else if (which && -lt - lga > 1.0) {
    double x = -lt - lga;
    x = fmax(-lt - lga + (a - 1.0) * log(x), 1.0);
    x = fmax(-lt - lga + (a - 1.0) * log(x), 1.0);
    u = log(x);
  }
  double lo = -745.2, hi = 709.8, dx = hi - lo, dold = dx;
  u = fmin(fmax(u, lo), hi);
  for (int it = 0; it < 64; ++it) {
    const double x = exp(u), lpref = a * u - x - lga;
    double e;
    const double g = sg * (ptk_gamma_logpq(a, x, lpref, which, &e) - lt);
    if (g == 0.0) break;
    if (g < 0.0) lo = u; else hi = u;
    // Halley's correction only while it is small (far from the root it is a difference of large terms)
    const double d = g / e, hf = 0.5 * d * (a - x - sg * e), tol = 2.0e-15 * fmax(1.0, fabs(u));
    double un = u - (fabs(hf) < 0.5 ? d / (1.0 - hf) : d);
    const bool inside = un >= lo && un <= hi;
    if (inside && fabs(d) <= tol) { u = un; break; }
    // bisect when the step leaves the bracket or does not halve the step before last, unless the Newton step has
    // stopped shrinking at the rounding noise of the forward function: then the root is found
    if (!inside || fabs(un - u) > 0.5 * fabs(dold)) {
      if (inside && fabs(d) < 1e-11 * fmax(1.0, fabs(u))) { u = un; break; }
      un = 0.5 * (lo + hi);
    }
    dold = dx;
    dx = un - u;
    u = un;
    if (hi - lo <= tol) break;
  }
  return exp(u);
}
__device__ inline double ptk_gammaincinv(double a, double p) {
  if (!(a > 0.0) || isinf(a) || !(p >= 0.0 && p <= 1.0)) return __longlong_as_double(0x7ff8000000000000LL);
  if (p == 0.0) return 0.0;
  if (p == 1.0) return __longlong_as_double(0x7ff0000000000000LL);
  return ptk_gammaincinv_tail(a, p, 0);
}
__device__ inline double ptk_gammainccinv(double a, double q) {
  if (!(a > 0.0) || isinf(a) || !(q >= 0.0 && q <= 1.0)) return __longlong_as_double(0x7ff8000000000000LL);
  if (q == 0.0) return __longlong_as_double(0x7ff0000000000000LL);
  if (q == 1.0) return 0.0;
  return ptk_gammaincinv_tail(a, q, 1);
}
#endif
""",
    # Inverse regularised incomplete beta (needs "betainc"), by the same scheme as "gammaincinv": the solver targets the
    # tail <= 1/2 (I_x(a,b) = p, or I_{1-x}(b,a) = 1-p through the a<->b, x<->1-x symmetry) and iterates on the logit
    # v = log(x / (1-x)), from which both x and 1-x follow to full relative precision.  log I is the log prefactor
    # a log x + b log(1-x) - log B(a,b) plus the log of ptk_betainc_cf over a (x <= (a+1)/(a+b+2)), or log1p of minus
    # the same form of I_{1-x}(b,a) (above): one formula family on both sides, so the residual has no jump where the
    # side changes.  Start: the normal approximation of AS 109 (Cran, Martin & Thomas 1977) for a, b > 1, else
    # x^a / (a B(a,b)) = p; then bracketed Halley steps on v in [-745.2, 745.2].  At most 64 iterations: worst case 64
    # continued-fraction evaluations (each capped at 300 terms, no other loop) per element.  Quantiles below DBL_MIN return the largest
    # denormal, as SciPy does in general (it returns 0 for b = 1, for a = b = 1/2 and for some denormal quantiles, see
    # DESIGN.md section 9).
    "betaincinv": r"""
#ifndef PTK_HAVE_BETAINCINV
#define PTK_HAVE_BETAINCINV
// log I_x(a, b), with x and xc = 1 - x both given to full precision (lx, lxc their logs) and lb = log B(a, b); *e gets
// d log I / d logit(x) = x^a (1-x)^b / (B(a,b) I).  Both sides use the same log prefactor and continued fraction:
// I_x(a, b) itself for x <= (a+1)/(a+b+2), 1 - I_{1-x}(b, a) above.  That switch keeps each fraction where it converges
// within its 300 terms (the mean a/(a+b) would not: at a = 4497, b = 1.2e-3 the root lies between 1 - (a+1)/(a+b+2)
// and the mean, where I_x(a, b)'s fraction has not converged), so log I is continuous across it to rounding and never
// passes through a linear-scale value that could overflow or underflow
__device__ inline double ptk_betainc_log(double a, double b, double x, double xc, double lx, double lxc, double lb,
                                         double* e) {
  const double lp = a * lx + b * lxc - lb;  // log of x^a (1-x)^b / B(a, b)
  if (x * (a + b + 2.0) <= a + 1.0) {
    const double w = (x * (a + b - 2.0) - (a - 1.0) < 0.0) ? ptk_betainc_cf(a, b, x, 0) : ptk_betainc_cf(a, b, x, 1) / xc;
    *e = a / w;
    return lp - log(a) + log(w);
  }
  const double w = (xc * (a + b - 2.0) - (b - 1.0) < 0.0) ? ptk_betainc_cf(b, a, xc, 0) : ptk_betainc_cf(b, a, xc, 1) / x;
  const double li = log1p(-exp(lp - log(b) + log(w)));
  *e = exp(lp - li);
  return li;
}
__device__ inline double ptk_betaincinv(double a, double b, double p) {
  // (SciPy's floor for an underflowing quantile is the largest denormal, one ulp below DBL_MIN)
  const double nan = __longlong_as_double(0x7ff8000000000000LL), largest_denormal = __longlong_as_double(0x000fffffffffffffLL);
  if (!(a > 0.0) || !(b > 0.0) || !(p >= 0.0 && p <= 1.0)) return nan;
  if (p == 0.0) return 0.0;
  if (p == 1.0) return 1.0;
  if (isinf(a)) return isinf(b) ? nan : 1.0;
  if (isinf(b)) return 0.0;
  int which = 0;
  double t = p;
  if (t > 0.5) { t = 1.0 - t; which = 1; }
  // solve for the lower tail of (A, B) at y, where y = x (which = 0) or y = 1 - x (which = 1); v is the logit of y
  const double A = which ? b : a, B = which ? a : b, lt = log(t);
  // log B(a, b); with the larger parameter L >= 20, lgamma(L) - lgamma(L + s) from Stirling's series, where
  // log1p keeps the digits lgamma's difference would cancel (s = 1e-3 next to L = 1e6)
  const double s = fmin(a, b), L = fmax(a, b);
  double lb = lgamma(a) + lgamma(b) - lgamma(a + b);
  if (L >= 20.0) {
    const double r = 1.0 / L, r2 = r * r, q = 1.0 / (L + s), q2 = q * q;
    const double cl = r * (0.08333333333333333 - r2 * (0.002777777777777778 - r2 * (7.936507936507937e-4 - r2 * 5.952380952380952e-4)));
    const double cq = q * (0.08333333333333333 - q2 * (0.002777777777777778 - q2 * (7.936507936507937e-4 - q2 * 5.952380952380952e-4)));
    lb = lgamma(s) - (L - 0.5) * log1p(s / L) - s * log(L + s) + s + (cl - cq);
  }
  double v = (lt + log(A) + lb) / A;  // log y from y^A / (A B(A,B)) = t
  if (!which && v < -708.3964185322641) return largest_denormal;
  if (A > 1.0 && B > 1.0) {
    const double r = sqrt(-2.0 * lt);
    const double y = r - (2.30753 + 0.27061 * r) / (1.0 + (0.99229 + 0.04481 * r) * r);
    const double h = 2.0 / (1.0 / (2.0 * A - 1.0) + 1.0 / (2.0 * B - 1.0)), lam = (y * y - 3.0) / 6.0;
    const double w = y * sqrt(h + lam) / h - (1.0 / (2.0 * B - 1.0) - 1.0 / (2.0 * A - 1.0)) * (lam + 5.0 / 6.0 - 2.0 / (3.0 * h));
    v = log(A / B) - 2.0 * w;
  } else {
    v = v - log1p(-exp(fmin(v, -1e-3)));
  }
  double lo = -745.2, hi = 745.2, dx = hi - lo, dold = dx;
  v = fmin(fmax(v, lo), hi);
  for (int it = 0; it < 64; ++it) {
    const double y = 1.0 / (1.0 + exp(-v)), yc = 1.0 / (1.0 + exp(v));
    const double ly = -log1p(exp(-v)), lyc = -log1p(exp(v));
    double e;
    const double g = ptk_betainc_log(A, B, y, yc, ly, lyc, lb, &e) - lt;
    if (g == 0.0) break;
    if (g < 0.0) lo = v; else hi = v;
    const double d = g / e, hf = 0.5 * d * (A * yc - B * y - e), tol = 2.0e-15 * fmax(1.0, fabs(v));
    double vn = v - (fabs(hf) < 0.5 ? d / (1.0 - hf) : d);
    const bool inside = vn >= lo && vn <= hi;
    if (inside && fabs(d) <= tol) { v = vn; break; }
    if (!inside || fabs(vn - v) > 0.5 * fabs(dold)) {
      if (inside && fabs(d) < 1e-11 * fmax(1.0, fabs(v))) { v = vn; break; }
      vn = 0.5 * (lo + hi);
    }
    dold = dx;
    dx = vn - v;
    v = vn;
    if (hi - lo <= tol) break;
  }
  const double x = which ? 1.0 / (1.0 + exp(v)) : 1.0 / (1.0 + exp(-v));
  return x < largest_denormal ? largest_denormal : x;
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
