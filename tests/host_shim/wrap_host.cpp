// Host build of the SHIPPED device function csdrb::wrap_phase_pm_pi (csdr_b200/csrc/common.cuh) for the CPU test tier:
// the CUDA intrinsics it uses are mapped onto the same IEEE-754 single-precision operations (SSE, no contraction), everything
// else in the header is never instantiated on the host.  Built and driven by tests/test_phase_wrap_host.py.
#include <cstdint>
#include <cstring>
#include <cmath>
#include <cuda_runtime.h>

static inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline size_t __cvta_generic_to_shared(const void*) { return 0; }
static inline int __float2int_rz(float f) { return (int)f; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }

#include "../../csdr_b200/csrc/common.cuh"
#include "../../csdr_b200/csrc/phase_table.cuh"

extern "C" {
// the reference's loop, libcsdr_gpl.c:49-50 (PI is the float constant of libcsdr.h:65); guarded like the device code for |ph| >= 2^26
float wrap_loop(float ph)
{
    const float PI = (float)3.14159265358979323846;
    if (!(std::fabs(ph) < 67108864.f)) return ph;
    while (ph > PI) { volatile float t = ph - 2 * PI; ph = t; }
    while (ph < -PI) { volatile float t = ph + 2 * PI; ph = t; }
    return ph;
}
float wrap_fast(float ph) { return csdrb::wrap_phase_pm_pi(ph); }
// returns the number of mismatches over n inputs (first mismatching input in *bad)
long wrap_compare(const float* x, long n, float* bad)
{
    long miss = 0;
    for (long i = 0; i < n; i++) {
        const float a = wrap_loop(x[i]), b = wrap_fast(x[i]);
        if (__float_as_uint(a) != __float_as_uint(b)) { if (!miss && bad) *bad = x[i]; miss++; }
    }
    return miss;
}

// ---- phase_table.cuh: the wrap as a table lookup for one fixed increment ---------------------------------------------------------------
// builds the table for `inc` and walks floats of its window (every `stride`-th one plus everything within 3 ulps of a threshold), both
// signs, comparing wrap_after_add with the loop.  Returns mismatches; *pieces = table size (0: no table -- the fallback is what runs);
// *checked = values compared.
long table_check(float inc, long stride, int* pieces, long* checked, float* bad)
{
    csdrb::WrapTable t;
    csdrb::wrap_table_build(inc, &t);
    *pieces = t.n; *checked = 0;
    long miss = 0;
    auto one = [&](float a) {
        for (int s = 0; s < 2; s++) {
            const float x = s ? -a : a;
            const float w = wrap_loop(x), g = csdrb::wrap_after_add(x, &t);
            if (__float_as_uint(w) != __float_as_uint(g)) { if (!miss && bad) *bad = x; miss++; }
            (*checked)++;
        }
    };
    const float ainc = std::fabs(inc);
    float lo = t.n ? t.lo : (ainc > 4.5f ? ainc - 4.5f : 0.f), hi = t.n ? t.hi : ainc + 4.5f;
    for (unsigned u = __float_as_uint(lo), e = __float_as_uint(hi); u <= e; u += (unsigned)stride) one(__uint_as_float(u));   // positive floats: +1 in the bits = next float
    for (int i = 0; i < t.n; i++) {
        float a = t.thr[i];
        for (int d = 0; d < 3; d++) a = std::nextafterf(a, 0.f);
        for (int d = 0; d < 7; d++) { if (a >= lo && a <= hi) one(a); a = std::nextafterf(a, INFINITY); }
    }
    one(std::nextafterf(lo, 0.f)); one(std::nextafterf(hi, INFINITY));            // just outside the window: the fallback path
    return miss;
}
// the chain itself: n steps of ph <- wrap(fl(ph + inc)) with the table and with the loop; returns the first step at which they differ (-1: never)
long table_chain(float inc, float ph0, long n)
{
    csdrb::WrapTable t;
    csdrb::wrap_table_build(inc, &t);
    float a = ph0, b = ph0;
    for (long i = 0; i < n; i++) {
        a = csdrb::wrap_after_add(__fadd_rn(a, inc), &t);
        b = wrap_loop(__fadd_rn(b, inc));
        if (__float_as_uint(a) != __float_as_uint(b)) return i;
    }
    return -1;
}
}
