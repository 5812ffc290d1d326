// TEST INFRASTRUCTURE ONLY — linked into oracle/_ref/libpbrt_ref.so, never into the product.
//
// The reference's float transcendentals, routed through this file by the linker: Makefile.ref links libpbrt_ref.so with
// -Wl,--wrap=sinf,--wrap=cosf,--wrap=sincosf,--wrap=logf,--wrap=atan2f,--wrap=acosf, so every call the reference's objects
// make to one of these six functions lands in the __wrap_ function of the same name below.  These six are exactly the float
// transcendentals that the path's reference units import (Beckmann's atanf / expf / powf / tanf aside, which the path does
// not reach).
//
// While ref_devmath_active (ref_harness.cpp) is 0, each wrapper is glibc's own function (__real_*), bit for bit.  While it
// is 1, each computes what the device computes: the double-precision routine rounded to float, written exactly as
// pbrt_v3_b200/csrc/device/pb2_math.cuh writes psinf / pcosf / psincosf / plogf / patan2f / pacosf.  The harness turns it on
// around evaluation only (ref_set_device_math), so the reference then differs from the CUDA path by nothing but the last
// bits of CUDA's double routines against glibc's, which lie far below float precision.
#include <atomic>
#include <math.h>

extern std::atomic<int> ref_devmath_active;

extern "C" {
float __real_sinf(float);
float __real_cosf(float);
void __real_sincosf(float, float *, float *);
float __real_logf(float);
float __real_atan2f(float, float);
float __real_acosf(float);

static inline bool deviceMath() { return ref_devmath_active.load(std::memory_order_relaxed) != 0; }

float __wrap_sinf(float x) {
    if (!deviceMath()) return __real_sinf(x);
    return (float)sin((double)x);
}
float __wrap_cosf(float x) {
    if (!deviceMath()) return __real_cosf(x);
    return (float)cos((double)x);
}
void __wrap_sincosf(float x, float *s, float *c) {
    if (!deviceMath()) {
        __real_sincosf(x, s, c);
        return;
    }
    double ds, dc;
    sincos((double)x, &ds, &dc);
    *s = (float)ds;
    *c = (float)dc;
}
float __wrap_logf(float x) {
    if (!deviceMath()) return __real_logf(x);
    return (float)log((double)x);
}
float __wrap_atan2f(float y, float x) {
    if (!deviceMath()) return __real_atan2f(y, x);
    return (float)atan2((double)y, (double)x);
}
float __wrap_acosf(float x) {
    if (!deviceMath()) return __real_acosf(x);
    return (float)acos((double)x);
}
}  // extern "C"
