// TEST INFRASTRUCTURE: the host spellings of the CUDA constructs that morefusion_b200/csrc/
// mesh_models.cu adds to those of mapping_emu_stubs.h (one thread at a time; compiled with
// -ffp-contract=off, as the .cu is built with -fmad=false).
#pragma once
#include <stdint.h>

using std::isfinite;
using std::max;

template <class T> static inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicXor(T* p, T v) { T o = *p; *p = o ^ v; return o; }
