// oracle/permutohedral/ref_capi.cpp -- TEST INFRASTRUCTURE: a C entry point into the reference's unmodified permutohedral
// lattice (third_party/permutohedral/permutohedral.cpp), for ctypes.  Written for this repository.
#include "permutohedral.h"

#define PRL_EXPORT extern "C" __attribute__((visibility("default")))

// Permutohedral::init over `feature` (n points x d, row-major) then compute() of `value` (n x vs, row-major) into `out` (n x vs),
// as probreg/gaussian_filtering.py does (filter(v, start) ignores start).  *lattice_size: getLatticeSize().
PRL_EXPORT int prl_filter(const float* feature, int n, int d, const float* value, int vs, int with_blur, float* out, int* lattice_size) {
    if (n < 1 || d < 1 || vs < 1) return -1;
    Eigen::MatrixXf f(d, n), v(vs, n), o(vs, n);
    for (int k = 0; k < n; ++k) {
        for (int j = 0; j < d; ++j) f(j, k) = feature[(size_t)k * d + j];
        for (int c = 0; c < vs; ++c) v(c, k) = value[(size_t)k * vs + c];
    }
    Permutohedral ph;
    ph.init(f, with_blur != 0);
    ph.compute(o, v);
    for (int k = 0; k < n; ++k)
        for (int c = 0; c < vs; ++c) out[(size_t)k * vs + c] = o(c, k);
    *lattice_size = ph.getLatticeSize();
    return 0;
}

// the lattice size alone (the E-step's blur / no-blur decision)
PRL_EXPORT int prl_lattice_size(const float* feature, int n, int d, int with_blur) {
    if (n < 1 || d < 1) return -1;
    Eigen::MatrixXf f(d, n);
    for (int k = 0; k < n; ++k)
        for (int j = 0; j < d; ++j) f(j, k) = feature[(size_t)k * d + j];
    Permutohedral ph;
    ph.init(f, with_blur != 0);
    return ph.getLatticeSize();
}
