// TEST INFRASTRUCTURE: the host spellings of the CUDA constructs that morefusion_b200/csrc/
// render_cad.cu adds to those of mapping_emu_stubs.h (one thread at a time; compiled with
// -ffp-contract=off, as the .cu is built with -fmad=false).
#pragma once
#include <stdint.h>

using std::isfinite;
using std::max;

struct int4 { int x, y, z, w; };
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
template <class T> static inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline float __double2float_rn(double a) { return (float)a; }
