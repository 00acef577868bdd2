// TEST INFRASTRUCTURE: the host spellings of the CUDA constructs that the render and box kernels
// of morefusion_b200/csrc/mapping.cu add to those of mapping_emu_stubs.h (one thread at a time,
// warps of one lane).
#pragma once

template <class T> static inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
// a group of one lane reduces to its own value
static inline unsigned __reduce_min_sync(unsigned, unsigned v) { return v; }
static inline unsigned __reduce_max_sync(unsigned, unsigned v) { return v; }
static inline unsigned __float_as_uint(float f) { unsigned u; __builtin_memcpy(&u, &f, 4); return u; }
