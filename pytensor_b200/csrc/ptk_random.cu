// Random draws on the device (SURVEY.md §8(f).3; reference: RandomVariable, pytensor/tensor/random/op.py:49, whose perform
// :457-468 calls numpy.random.Generator methods on the host).  numpy's PCG64 stream with its rejection samplers is inherently
// sequential; here every output element owns a COUNTER-BASED stream instead: Philox4x32-10 keyed by 128 bits the caller
// takes from the host Generator (which thereby advances), counter = (element index, draw round).  Same seed => same
// draws, any element computable independently, no state in device memory.  Values therefore differ from the C linker's;
// parity is distributional (moments + Kolmogorov-Smirnov in tests/test_gpu_random.py), shapes / dtypes / the
// advance-the-generator contract are exact.
#include <math.h>
#include <algorithm>
#include "ptk_common.h"

namespace {

using ptk::fail;

struct Philox {
  uint32_t k0, k1;
  __device__ __forceinline__ void round(uint32_t (&c)[4], uint32_t ka, uint32_t kb) const {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
    const uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
    const uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ ka, n1 = lo1, n2 = hi0 ^ c[3] ^ kb, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  }
  __device__ __forceinline__ void block(uint32_t (&c)[4]) const {
    uint32_t ka = k0, kb = k1;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      round(c, ka, kb);
      ka += 0x9E3779B9u;
      kb += 0xBB67AE85u;
    }
  }
};

// 53-bit uniforms in (0, 1): never 0, never 1 (safe for log / tan)
__device__ __forceinline__ double u01(uint32_t hi, uint32_t lo) {
  const uint64_t b = (((uint64_t)hi << 32) | lo) >> 11;
  return ((double)b + 0.5) * (1.0 / 9007199254740992.0);
}

__device__ __forceinline__ double ptk_tanpi(double t) { return sinpi(t) / cospi(t); }

struct Draws {   // counter-based supply of uniforms / normals for ONE output element
  Philox ph;
  uint64_t idx, seed_hi;
  uint32_t round_;
  uint32_t c[4];
  int have;
  __device__ __forceinline__ Draws(uint64_t k, uint64_t s, uint64_t i) : idx(i), seed_hi(s), round_(0), have(0) {
    ph.k0 = (uint32_t)k;
    ph.k1 = (uint32_t)(k >> 32);
  }
  __device__ __forceinline__ double uniform() {
    if (have == 0) {
      c[0] = (uint32_t)idx; c[1] = (uint32_t)(idx >> 32); c[2] = round_++ ^ (uint32_t)seed_hi; c[3] = (uint32_t)(seed_hi >> 32);
      ph.block(c);
      have = 2;
    }
    --have;
    return have == 1 ? u01(c[0], c[1]) : u01(c[2], c[3]);
  }
  __device__ __forceinline__ double normal() {   // Box-Muller, one of the pair
    const double u = uniform(), v = uniform();
    return sqrt(-2.0 * log(u)) * cospi(2.0 * v);
  }
  __device__ double gamma(double a) {            // Marsaglia & Tsang (2000); a < 1 through the a+1 boost
    if (!(a > 0.0)) return a == 0.0 ? 0.0 : __longlong_as_double(0x7ff8000000000000LL);
    double boost = 1.0;
    if (a < 1.0) {
      boost = pow(uniform(), 1.0 / a);
      a += 1.0;
    }
    const double d = a - 1.0 / 3.0, cc = 1.0 / sqrt(9.0 * d);
    for (int it = 0; it < 64; ++it) {
      const double x = normal();
      double v = 1.0 + cc * x;
      if (v <= 0.0) continue;
      v = v * v * v;
      const double u = uniform();
      if (u < 1.0 - 0.0331 * (x * x) * (x * x) || log(u) < 0.5 * x * x + d * (1.0 - v + log(v))) return boost * d * v;
    }
    return boost * d;
  }
  __device__ double log_gamma(double a) {        // log of a gamma(a) draw: the a < 1 boost as log(u) / a, so tiny shapes
    if (!(a > 0.0)) return a == 0.0 ? -HUGE_VAL : __longlong_as_double(0x7ff8000000000000LL);   // do not underflow to 0
    double lboost = 0.0;
    if (a < 1.0) {
      lboost = log(uniform()) / a;
      a += 1.0;
    }
    const double d = a - 1.0 / 3.0, cc = 1.0 / sqrt(9.0 * d);
    for (int it = 0; it < 64; ++it) {            // the cap of gamma()
      const double x = normal();
      double v = 1.0 + cc * x;
      if (v <= 0.0) continue;
      v = v * v * v;
      const double u = uniform();
      if (u < 1.0 - 0.0331 * (x * x) * (x * x) || log(u) < 0.5 * x * x + d * (1.0 - v + log(v))) return lboost + log(d * v);
    }
    return lboost + log(d);
  }
  __device__ double beta(double a, double b) {   // a, b > 0; through log-gammas, so a + b << 1 still gives a value in [0, 1]
    const double la = log_gamma(a), lb = log_gamma(b);
    return 1.0 / (1.0 + exp(lb - la));
  }

  // Poisson(lam), 0 <= lam <= POISSON_LAM_MAX.
  //  lam < 10: inversion with one uniform, a sequential search of the cdf that stops when a term no longer changes it
  //    (after at most ~50 terms; 256 caps it).
  //  lam >= 10: PTRS transformed rejection (Hormann 1993).  Each round accepts with probability > 0.89, so the cap of 64
  //    rounds is reached with probability < 1e-61; floor(lam) is returned then.
  __device__ double poisson(double lam) {
    if (lam < 10.0) {
      const double u = uniform();
      double t = exp(-lam), F = t, k = 0.0;
      for (int it = 0; it < 256 && u > F; ++it) {
        k += 1.0;
        t *= lam / k;
        if (F + t == F) break;
        F += t;
      }
      return k;
    }
    const double slam = sqrt(lam), loglam = log(lam), b = 0.931 + 2.53 * slam, a = -0.059 + 0.02483 * b;
    const double inv_alpha = 1.1239 + 1.1328 / (b - 3.4), vr = 0.9277 - 3.6224 / (b - 2.0);
    // log pmf(k) = (k - lam) log(lam) + c0 - [lgamma(k + 1) - lgamma(lam + 1)], c0 = lam log(lam) - lam - lgamma(lam + 1),
    // both without the cancellation of terms ~lam log(lam) (lam reaches 9.2e18)
    const double c0 = lam >= 16.0 ? -lam * log1p(1.0 / lam) - 0.5 * log(lam + 1.0) + 1.0 - 0.91893853320467274 - stirling_tail(lam + 1.0)
                                  : lam * loglam - lam - lgamma(lam + 1.0);
    for (int it = 0; it < 64; ++it) {
      const double U = uniform() - 0.5, V = uniform(), us = 0.5 - fabs(U);
      const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
      if (us >= 0.07 && V <= vr) return k;
      if (k < 0.0 || (us < 0.013 && V > us)) continue;
      if (log(V * inv_alpha / (a / (us * us) + b)) <= (k - lam) * loglam + c0 - lgamma_diff(k + 1.0, lam + 1.0)) return k;
    }
    return floor(lam);
  }

  // Binomial(n, p), n a non-negative integer below 2^53, 0 <= p <= 1; p > 1/2 through the symmetry n - Binomial(n, 1 - p).
  //  n p < 10: inversion with one uniform (a sequential search of the cdf, stopping as poisson() does).
  //  otherwise: BTRS transformed rejection (Hormann 1993), capped at 64 rounds like poisson(); the mode is returned then.
  __device__ double binomial(double n, double p) {
    if (n == 0.0 || p == 0.0) return 0.0;
    const bool flip = p > 0.5;
    const double pp = flip ? 1.0 - p : p, q = 1.0 - pp;
    double k = 0.0;
    if (n * pp < 10.0) {
      const double u = uniform(), r = pp / q;
      double t = exp(n * log1p(-pp)), F = t;
      for (int it = 0; it < 256 && u > F && k < n; ++it) {
        t *= r * (n - k) / (k + 1.0);
        k += 1.0;
        if (F + t == F) break;
        F += t;
      }
    } else {
      const double spq = sqrt(n * pp * q), b = 1.15 + 2.53 * spq, a = -0.0873 + 0.0248 * b + 0.01 * pp, c = n * pp + 0.5;
      const double alpha = (2.83 + 5.1 / b) * spq, vr = 0.92 - 4.2 / b, m = floor((n + 1.0) * pp), lpq = log(pp / q);
      k = m;
      for (int it = 0; it < 64; ++it) {
        const double U = uniform() - 0.5, V = uniform(), us = 0.5 - fabs(U);
        const double kk = floor((2.0 * a / us + b) * U + c);
        if (kk < 0.0 || kk > n) continue;
        if ((us >= 0.07 && V <= vr) ||
            log(V * alpha / (a / (us * us) + b)) <=
                lgamma_diff(m + 1.0, kk + 1.0) + lgamma_diff(n - m + 1.0, n - kk + 1.0) + (kk - m) * lpq) {
          k = kk;
          break;
        }
      }
    }
    return flip ? n - k : k;
  }

  // Geometric(p), 0 < p <= 1, support from 1: ceil(log(u) / log1p(-p)) (NumPy clamps at 2^63 - 1: count_out does)
  __device__ double geometric(double p) {
    if (p >= 1.0) return 1.0;
    return fmax(1.0, ceil(log(uniform()) / log1p(-p)));
  }

  // Stirling-series helpers of the rejection tests
  __device__ static double stirling_tail(double z) {   // lgamma(z) - [(z - 1/2) log z - z + log(2 pi) / 2], z >= 16
    const double r = 1.0 / (z * z);
    return (1.0 / 12.0 - r * (1.0 / 360.0 - r / 1260.0)) / z;
  }
  __device__ static double lgamma_diff(double x, double y) {   // lgamma(x) - lgamma(y), x, y >= 1, accurate when both are large
    if (x < 16.0 || y < 16.0) return lgamma(x) - lgamma(y);
    const double d = x - y;
    return (x - 0.5) * log1p(d / y) + d * (log(y) - 1.0) + stirling_tail(x) - stirling_tail(y);
  }
};

enum Dist { UNIFORM = 0, NORMAL = 1, HALFNORMAL = 2, LOGNORMAL = 3, EXPONENTIAL = 4, LAPLACE = 5, LOGISTIC = 6, GUMBEL = 7,
            CAUCHY = 8, BERNOULLI = 9, GAMMA = 10, BETA = 11, INTEGERS = 12, WEIBULL = 13, PARETO = 14, HALFCAUCHY = 15,
            INVGAMMA = 16, STUDENTT = 17, N_DIST = 18 };

template <typename OUT>
__global__ void __launch_bounds__(256) random_kernel(int dist, OUT* __restrict__ out, long long n, uint64_t key, uint64_t seed,
                                                     const double* __restrict__ p0, long long s0,
                                                     const double* __restrict__ p1, long long s1,
                                                     const double* __restrict__ p2, long long s2) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    Draws g(key, seed, (uint64_t)i);
    const double a = p0 ? p0[i * s0] : 0.0, b = p1 ? p1[i * s1] : 1.0, c = p2 ? p2[i * s2] : 1.0;
    double x;
    switch (dist) {
      case UNIFORM: x = a + (b - a) * g.uniform(); break;
      case NORMAL: x = a + b * g.normal(); break;
      case HALFNORMAL: x = a + b * fabs(g.normal()); break;
      case LOGNORMAL: x = exp(a + b * g.normal()); break;
      case EXPONENTIAL: x = -a * log(g.uniform()); break;                       // a = scale
      case LAPLACE: { const double u = g.uniform() - 0.5; x = a - b * copysign(log(1.0 - 2.0 * fabs(u)), u); } break;
      case LOGISTIC: { const double u = g.uniform(); x = a + b * log(u / (1.0 - u)); } break;
      case GUMBEL: x = a - b * log(-log(g.uniform())); break;
      case CAUCHY: x = a + b * ptk_tanpi(g.uniform() - 0.5); break;
      case HALFCAUCHY: x = a + b * fabs(ptk_tanpi(g.uniform() - 0.5)); break;
      case BERNOULLI: x = g.uniform() < a ? 1.0 : 0.0; break;                    // a = p
      case GAMMA: x = b * g.gamma(a); break;                                     // a = shape, b = scale
      case INVGAMMA: x = b / g.gamma(a); break;                                  // a = shape, b = scale
      case BETA: { const double ga = g.gamma(a), gb = g.gamma(b); x = ga / (ga + gb); } break;
      case INTEGERS: x = floor(a + (b - a) * g.uniform()); if (x >= b) x = b - 1.0; break;   // [low, high)
      case WEIBULL: x = pow(-log(g.uniform()), 1.0 / a); break;                  // a = shape
      case PARETO: x = b * pow(g.uniform(), -1.0 / a); break;                    // scipy's form (x >= scale), a = shape, b = scale
      case STUDENTT: { const double z = g.normal(), ch = 2.0 * g.gamma(0.5 * a); x = b + c * z / sqrt(ch / a); } break;  // a=df
      default: x = 0.0;
    }
    out[i] = (OUT)x;
  }
}

// ---- discrete counts and row samplers ------------------------------------------------------------------------------------
// Parameters the reference rejects (NumPy's Generator / SciPy's argcheck) set the launch's error word to 1 and leave a 0
// draw; the caller raises ValueError.  Every writer stores the same value, so a plain store is enough.
enum CountDist { POISSON = 0, BINOMIAL = 1, NEGATIVE_BINOMIAL = 2, GEOMETRIC = 3, BETA_BINOMIAL = 4, N_COUNT = 5 };

constexpr double POISSON_LAM_MAX = 9.2233720064847708e18;   // NumPy's: int64 max - 10 sqrt(int64 max)
constexpr double EXACT_INT_MAX = 9007199254740992.0;        // 2^53: larger integer n do not survive the float64 parameters

template <typename OUT>
__device__ __forceinline__ OUT count_out(double x) {         // int64 saturates at 2^63 - 1 (NumPy's geometric)
  return x >= 9223372036854775807.0 ? (OUT)(long long)0x7fffffffffffffffLL : (OUT)(long long)x;
}

template <typename OUT>
__global__ void __launch_bounds__(256) count_kernel(int dist, OUT* __restrict__ out, long long n, uint64_t key, uint64_t seed,
                                                    const double* __restrict__ p0, long long s0,
                                                    const double* __restrict__ p1, long long s1,
                                                    const double* __restrict__ p2, long long s2, int* __restrict__ err) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    Draws g(key, seed, (uint64_t)i);
    const double a = p0 ? p0[i * s0] : 0.0, b = p1 ? p1[i * s1] : 1.0, c = p2 ? p2[i * s2] : 1.0;
    double x = 0.0;
    bool ok = false;
    switch (dist) {
      case POISSON:                                                              // a = lam
        ok = a >= 0.0 && a <= POISSON_LAM_MAX;
        if (ok) x = g.poisson(a);
        break;
      case BINOMIAL:                                                             // a = n, b = p
        ok = a >= 0.0 && a <= EXACT_INT_MAX && b >= 0.0 && b <= 1.0;
        if (ok) x = g.binomial(a, b);
        break;
      case NEGATIVE_BINOMIAL:                                                    // a = n, b = p; Poisson(Gamma(n, (1-p)/p))
        ok = a > 0.0 && b > 0.0 && b <= 1.0 && (1.0 - b) / b * (a + 10.0 * sqrt(a)) <= POISSON_LAM_MAX;
        if (ok) x = g.poisson(fmin(g.gamma(a) * ((1.0 - b) / b), POISSON_LAM_MAX));
        break;
      case GEOMETRIC:                                                            // a = p
        ok = a > 0.0 && a <= 1.0;
        if (ok) x = g.geometric(a);
        break;
      case BETA_BINOMIAL:                                                        // a = n, b = alpha, c = beta
        ok = a >= 0.0 && a <= EXACT_INT_MAX && a == floor(a) && b > 0.0 && c > 0.0;
        if (ok) x = g.binomial(a, g.beta(b, c));
        break;
      default: break;
    }
    if (!ok) *err = 1;
    out[i] = count_out<OUT>(x);
  }
}

// Multinomial, one thread per row (stream = row): conditional binomials over categories 0..k-2, the last category takes the
// remainder whatever p[k-1] is (NumPy's algorithm).  p: row r at p + r * ps; n: nv[r * ns], truncated toward zero as the
// reference's batched rows convert a float n.
template <typename OUT>
__global__ void __launch_bounds__(256) multinomial_kernel(OUT* __restrict__ out, long long rows, long long k, uint64_t key,
                                                          uint64_t seed, const double* __restrict__ p, long long ps,
                                                          const double* __restrict__ nv, long long ns, int* __restrict__ err) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const double* pr = p + r * ps;
    OUT* o = out + r * k;
    const double n = trunc(nv[r * ns]);
    bool ok = n >= 0.0 && n <= EXACT_INT_MAX;
    double head = 0.0;                                                           // sum(p[:-1]); NumPy allows 1e-12 of slack
    for (long long j = 0; j < k; ++j) {
      const double pj = pr[j];
      ok = ok && pj >= 0.0 && pj <= 1.0;
      if (j < k - 1) head += pj;
    }
    if (!(ok && head <= 1.0 + 1e-12)) {
      *err = 1;
      for (long long j = 0; j < k; ++j) o[j] = (OUT)0;
      continue;
    }
    Draws g(key, seed, (uint64_t)r);
    double left = n, rest = 1.0;                                                 // trials left, probability mass left
    for (long long j = 0; j < k - 1; ++j) {
      const double x = left > 0.0 ? g.binomial(left, fmin(fmax(pr[j] / rest, 0.0), 1.0)) : 0.0;
      o[j] = (OUT)(long long)x;
      left -= x;
      rest -= pr[j];
    }
    if (k > 0) o[k - 1] = (OUT)(long long)left;
  }
}

}  // namespace

// ---- warp-per-row samplers (shuffles: kept out of the span above, which also compiles for the host) -------------------------
namespace {

constexpr unsigned FULL = 0xffffffffu;

// Categorical: one uniform per row (stream = row); the draw is the number of cumulative sums below u, i.e. NumPy's
// searchsorted(cumsum(p), u, side="left"), and k when u exceeds the total.  Lanes stride the categories 32 at a time with an
// fp64 warp scan carried across chunks.  A category with p == 0 must never be drawn whatever the summation order, so the
// test runs on a running maximum of the cumulative sums at nonzero categories: it is monotone, and equal across a zero.
template <typename OUT>
__global__ void __launch_bounds__(256) categorical_kernel(OUT* __restrict__ out, long long rows, long long k, uint64_t key,
                                                          uint64_t seed, const double* __restrict__ p, long long ps) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps) {
    Draws g(key, seed, (uint64_t)r);
    const double u = g.uniform();
    const double* pr = p + r * ps;
    double sum = 0.0, top = -HUGE_VAL;       // cumulative sum so far; the running maximum so far
    long long below = 0;
    for (long long j0 = 0; j0 < k && top < u; j0 += 32) {   // (warp-uniform: once top >= u no later sum counts)
      const long long j = j0 + lane;
      const double pj = j < k ? pr[j] : 0.0;
      double cs = pj;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const double t = __shfl_up_sync(FULL, cs, d);
        if (lane >= d) cs += t;
      }
      cs += sum;
      double m = pj != 0.0 ? cs : -HUGE_VAL;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const double t = __shfl_up_sync(FULL, m, d);
        if (lane >= d) m = fmax(m, t);
      }
      m = fmax(m, top);
      below += __popc(__ballot_sync(FULL, j < k && m < u));
      sum = __shfl_sync(FULL, cs, 31);
      top = __shfl_sync(FULL, m, 31);
    }
    if (lane == 0) out[r] = (OUT)below;
  }
}

// Dirichlet: one gamma per component (stream = row * k + j), in log space with a max-subtraction so that alpha ~ 1e-3, whose
// direct gamma draws underflow to 0, still gives a finite row summing to 1.  Pass 1 keeps a running (max, sum of exp) per
// lane, combined over the warp; pass 2 redraws each component from its stream and writes exp(l - max) / sum.
// alpha = 0 gives a 0 component (all zero: a 0 row), a NaN alpha a NaN row, alpha < 0 the error word.
template <typename OUT>
__global__ void __launch_bounds__(256) dirichlet_kernel(OUT* __restrict__ out, long long rows, long long k, uint64_t key,
                                                        uint64_t seed, const double* __restrict__ alpha, long long as,
                                                        int* __restrict__ err) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps) {
    const double* ar = alpha + r * as;
    double mx = -HUGE_VAL, s = 0.0;
    int flags = 0;                            // 1: an alpha < 0, 2: a NaN alpha
    for (long long j = lane; j < k; j += 32) {
      const double a = ar[j];
      flags |= (a < 0.0 ? 1 : 0) | (a != a ? 2 : 0);
      Draws g(key, seed, (uint64_t)(r * k + j));
      const double l = g.log_gamma(a);
      if (l > mx) {
        s = s * exp(mx - l) + 1.0;
        mx = l;
      } else if (l > -HUGE_VAL) {
        s += exp(l - mx);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const double om = __shfl_xor_sync(FULL, mx, d), os = __shfl_xor_sync(FULL, s, d);
      flags |= __shfl_xor_sync(FULL, flags, d);
      const double m = fmax(mx, om);
      s = (mx > -HUGE_VAL ? s * exp(mx - m) : 0.0) + (om > -HUGE_VAL ? os * exp(om - m) : 0.0);
      mx = m;
    }
    if ((flags & 1) && lane == 0) *err = 1;
    for (long long j = lane; j < k; j += 32) {
      double x;
      if (flags & 1) {
        x = 0.0;
      } else if (flags & 2) {
        x = __longlong_as_double(0x7ff8000000000000LL);
      } else if (!(mx > -HUGE_VAL)) {
        x = 0.0;
      } else {
        Draws g(key, seed, (uint64_t)(r * k + j));
        x = exp(g.log_gamma(ar[j]) - mx) / s;
      }
      out[r * k + j] = (OUT)x;
    }
  }
}

}  // namespace

extern "C" ptk_status ptk_random_fill(int dist, int dtype, void* out, int64_t n, uint64_t key, uint64_t seed, const void* p0,
                                      int64_t s0, const void* p1, int64_t s1, const void* p2, int64_t s2, void* stream) {
  PTK_REQUIRE_INIT();
  if (dist < 0 || dist >= N_DIST) return fail(PTK_ERR_ARG, "ptk_random_fill: unknown distribution");
  if (n <= 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned g = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)ptk::sm_count() * 16));
#define PTK_RND(T) random_kernel<T><<<g, 256, 0, st>>>(dist, (T*)out, n, key, seed, (const double*)p0, s0, (const double*)p1, s1, (const double*)p2, s2); break;
  switch (dtype) {
    case PTK_F32: PTK_RND(float)
    case PTK_F64: PTK_RND(double)
    case PTK_I64: PTK_RND(int64_t)
    case PTK_I32: PTK_RND(int32_t)
    case PTK_I16: PTK_RND(int16_t)
    case PTK_I8: PTK_RND(int8_t)
    case PTK_U8: case PTK_BOOL: PTK_RND(uint8_t)
    default: return fail(PTK_ERR_UNSUPPORTED, "ptk_random_fill: output dtype");
  }
#undef PTK_RND
  PTK_LAUNCH_CHECK("random_fill");
  return PTK_OK;
}

extern "C" ptk_status ptk_random_count(int dist, int dtype, void* out, int64_t n, uint64_t key, uint64_t seed, const void* p0,
                                       int64_t s0, const void* p1, int64_t s1, const void* p2, int64_t s2, int* err,
                                       void* stream) {
  PTK_REQUIRE_INIT();
  if (dist < 0 || dist >= N_COUNT) return fail(PTK_ERR_ARG, "ptk_random_count: unknown distribution");
  if (!err) return fail(PTK_ERR_ARG, "ptk_random_count: no error word");
  if (n <= 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned g = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)ptk::sm_count() * 16));
#define PTK_CNT(T) count_kernel<T><<<g, 256, 0, st>>>(dist, (T*)out, n, key, seed, (const double*)p0, s0, (const double*)p1, s1, (const double*)p2, s2, err); break;
  switch (dtype) {
    case PTK_F32: PTK_CNT(float)
    case PTK_F64: PTK_CNT(double)
    case PTK_I64: PTK_CNT(int64_t)
    case PTK_I32: PTK_CNT(int32_t)
    case PTK_I16: PTK_CNT(int16_t)
    case PTK_I8: PTK_CNT(int8_t)
    case PTK_U8: case PTK_BOOL: PTK_CNT(uint8_t)
    default: return fail(PTK_ERR_UNSUPPORTED, "ptk_random_count: output dtype");
  }
#undef PTK_CNT
  PTK_LAUNCH_CHECK("random_count");
  return PTK_OK;
}

extern "C" ptk_status ptk_random_rows(int kind, int dtype, void* out, int64_t rows, int64_t k, uint64_t key, uint64_t seed,
                                      const void* p, int64_t ps, const void* nv, int64_t ns, int* err, void* stream) {
  PTK_REQUIRE_INIT();
  if (kind < 0 || kind > 2) return fail(PTK_ERR_ARG, "ptk_random_rows: unknown sampler");
  if (!err || (kind == 1 && !nv)) return fail(PTK_ERR_ARG, "ptk_random_rows: missing error word or n");
  if (rows <= 0 || (kind != 0 && k <= 0)) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cap = (int64_t)ptk::sm_count() * 16;
  const unsigned gt = (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 255) / 256, cap));   // thread per row
  const unsigned gw = (unsigned)std::max<int64_t>(1, std::min<int64_t>((rows + 7) / 8, cap));       // warp per row
  const double* pd = (const double*)p;
#define PTK_ROWS(T)                                                                                                      \
  if (kind == 0) categorical_kernel<T><<<gw, 256, 0, st>>>((T*)out, rows, k, key, seed, pd, ps);                         \
  else if (kind == 1) multinomial_kernel<T><<<gt, 256, 0, st>>>((T*)out, rows, k, key, seed, pd, ps, (const double*)nv, ns, err); \
  else dirichlet_kernel<T><<<gw, 256, 0, st>>>((T*)out, rows, k, key, seed, pd, ps, err);                                 \
  break;
  switch (dtype) {
    case PTK_F32: PTK_ROWS(float)
    case PTK_F64: PTK_ROWS(double)
    case PTK_I64: PTK_ROWS(int64_t)
    case PTK_I32: PTK_ROWS(int32_t)
    case PTK_I16: PTK_ROWS(int16_t)
    case PTK_I8: PTK_ROWS(int8_t)
    case PTK_U8: case PTK_BOOL: PTK_ROWS(uint8_t)
    default: return fail(PTK_ERR_UNSUPPORTED, "ptk_random_rows: output dtype");
  }
#undef PTK_ROWS
  PTK_LAUNCH_CHECK("random_rows");
  return PTK_OK;
}
