// numpy's pairwise summation of a contiguous float64 array (np.sum / np.mean's reduction), restated for one device
// thread, and np.maximum / np.minimum of two doubles.  Shared by the evaluations whose results are graded byte-equal
// with numpy: include it only in translation units built with -fmad=false.
#pragma once

namespace {

// np.maximum / np.minimum: a NaN operand is the result (a when both are); otherwise the larger / smaller, and b when
// they compare equal (np.maximum(-0.0, 0.0) is 0.0).  A NaN b fails the compare and is returned.
__device__ __forceinline__ double np_max(double a, double b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ double np_min(double a, double b) { return (a != a || a < b) ? a : b; }

constexpr int kPwBlock = 128;  // numpy's PW_BLOCKSIZE
constexpr int kPwDepth = 48;

// one leaf of numpy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src): n < 8 in order from 0.; n <= 128 in
// eight interleaved accumulators, combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest in order
__device__ double pairwise_leaf(const double* a, long n) {
  if (n < 8) {
    double res = 0.0;
    for (long i = 0; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  long i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, a[i]);
  return res;
}

// np.sum of a contiguous float64 array: 0. + pairwise_sum(a, n), where above 128 elements the array splits at
// n2 = n / 2 rounded down to a multiple of 8 and the halves' sums are added.  Evaluated without recursion.
__device__ double np_sum(const double* a, long n) {
  long lo_s[kPwDepth], n_s[kPwDepth];
  double left_s[kPwDepth];
  int st_s[kPwDepth];
  int sp = 0;
  lo_s[0] = 0; n_s[0] = n; st_s[0] = 0;
  double ret = 0.0;
  while (sp >= 0) {
    const long lo = lo_s[sp], nn = n_s[sp];
    if (nn <= kPwBlock) {
      ret = pairwise_leaf(a + lo, nn);
      --sp;
      continue;
    }
    long n2 = nn / 2;
    n2 -= n2 % 8;
    if (st_s[sp] == 0) {
      st_s[sp] = 1;
      ++sp; lo_s[sp] = lo; n_s[sp] = n2; st_s[sp] = 0;
    } else if (st_s[sp] == 1) {
      left_s[sp] = ret;
      st_s[sp] = 2;
      ++sp; lo_s[sp] = lo + n2; n_s[sp] = nn - n2; st_s[sp] = 0;
    } else {
      ret = __dadd_rn(left_s[sp], ret);
      --sp;
    }
  }
  return __dadd_rn(0.0, ret);
}

}  // namespace
