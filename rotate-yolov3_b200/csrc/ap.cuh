// Per-class precision, recall, AP and F1 of ap_per_class / compute_ap (reference utils/utils.py:200-286) from the
// positions of one class's true positives among its confidence-sorted rows.  Shared by ap.cu and the host build the CPU
// tests compile with g++ (the way riou_area.cuh and jpeg.cuh are), so both evaluate the same float64 operations in the
// same order; products and sums go through ap_mul / ap_add so that nvcc cannot contract them into FMAs.
//
// Why the true positives suffice: within a class, recall only changes at a true positive, so compute_ap's sum has one
// term per true positive (plus (1 - r) * 0 at the end sentinel); between two true positives the precision
// tpc / (tpc + fpc) only falls, so the running maximum from the end, taken at a true positive, is the maximum over the
// true positives from there on.
#pragma once

#ifdef __CUDACC__
#define RY_AP_HD __host__ __device__ __forceinline__
#else
#define RY_AP_HD static inline
#endif

namespace ryolo {

#if defined(__CUDA_ARCH__)
RY_AP_HD double ap_mul(double a, double b) { return __dmul_rn(a, b); }
RY_AP_HD double ap_add(double a, double b) { return __dadd_rn(a, b); }
#else
RY_AP_HD double ap_mul(double a, double b) { return a * b; }
RY_AP_HD double ap_add(double a, double b) { return a + b; }
#endif

struct ApClass {
  double p, r, ap, f1;
};

// tp_pos[m] - first: position of the class's m-th true positive among its n_p rows sorted by confidence (ascending in m);
// n_gt > 0 targets of the class; env: ntp doubles of scratch.  n_p == 0 gives 0 / 0 / 0 / 0 like the reference.
RY_AP_HD ApClass ap_class_stats(const int* tp_pos, int first, int ntp, long long n_p, long long n_gt, double* env) {
  ApClass s;
  const double den = ap_add((double)n_gt, 1e-16);                          // n_gt + 1e-16
  s.p = n_p > 0 ? (double)ntp / (double)n_p : 0.0;                         // precision[-1] = tpc / (tpc + fpc)
  s.r = n_p > 0 ? (double)ntp / den : 0.0;                                 // recall[-1]
  double e = 0.0;                                                          // envelope: running max from the end
  for (int m = ntp - 1; m >= 0; m--) {
    const double prec = (double)(m + 1) / (double)(tp_pos[m] - first + 1);
    e = prec > e ? prec : e;
    env[m] = e;
  }
  double ap = 0.0, prev = 0.0;                                             // sum of delta recall * envelope, in row order
  for (int m = 0; m < ntp; m++) {
    const double rec = (double)(m + 1) / den;
    ap = ap_add(ap, ap_mul(rec - prev, env[m]));
    prev = rec;
  }
  s.ap = ap;
  s.f1 = ap_mul(ap_mul(2.0, s.p), s.r) / ap_add(ap_add(s.p, s.r), 1e-16);
  return s;
}

}  // namespace ryolo
