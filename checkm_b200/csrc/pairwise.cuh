// pairwise.cuh -- numpy's pairwise order for np.sum of a contiguous float64 vector, shared by the outlier scores
// (outliers.cu) and the plot windows (windows.cu).
//
// Below 8 elements a loop from 0.0; up to 128 elements (PW_LEAF, numpy's PW_BLOCKSIZE) eight running sums r[j] += a[i+j]
// combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), the tail added one by one; above 128 the vector is halved, the first
// half rounded down to a multiple of 8, and the halves' sums added.  oracle/outliers_oracle.py states the same and
// tests/test_outliers_cpu.py holds it to the installed numpy.
#pragma once
#include <set>

namespace ckm {

constexpr int PW_LEAF = 128;

// the sum of a leaf (n <= PW_LEAF elements) in numpy's order; a(i) returns element i
template <class A>
__device__ __forceinline__ double pw_leaf_sum(A a, int n) {
  if (n < 8) {
    double res = 0.0;
    for (int i = 0; i < n; ++i) res += a(i);
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = a(j);
  int i = 8;
  for (; i < n - n % 8; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] += a(i + j);
  }
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += a(i);
  return res;
}

// where numpy splits n > PW_LEAF elements: the first half's length
__host__ __device__ __forceinline__ long long pw_split(long long n) {
  long long n2 = n / 2;
  return n2 - n2 % 8;
}

// depth of numpy's pairwise tree over n elements
inline int pairwise_depth(long long n) {
  std::set<long long> level{n};
  int depth = 0;
  for (;;) {
    std::set<long long> next;
    for (long long c : level)
      if (c > PW_LEAF) { const long long n2 = pw_split(c); next.insert(n2); next.insert(c - n2); }
    if (next.empty()) return depth;
    level.swap(next);
    ++depth;
  }
}

}  // namespace ckm
