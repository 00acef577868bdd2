// average_voxelization_3d / max_voxelization_3d for sm_90a.
//
// Replaces the reference's CuPy kernels K1-K4 (SURVEY.md 2.2):
//   morefusion/functions/geometry/average_voxelization_3d.py:57-115, :163-218
//   morefusion/functions/geometry/max_voxelization_3d.py:75-138, :153-183
//
// average_voxelization_3d forward = two launches, no memsets, no atomics on HBM:
//   k_avg_prepass  one thread per point: voxel key, batch-segment boundaries, per-CTA flag word
//   k_avg_fused    a CTA owns (batch b, 1024 consecutive voxels, <= 64 channels).  It finds the
//                  points of b that fall into its voxels (ordered compaction of the keys), sums
//                  them per occupied voxel in ascending point order in shared memory, divides,
//                  and then streams its 4 KiB piece of every channel plane: one 16-byte store per
//                  thread and plane, zeros straight from registers, occupied voxels patched in
//                  from shared memory.  Every output element is written exactly once, so the
//                  operator costs one pass over the (mostly zero) dense output.
// Per-voxel sums are taken in ascending point order -> bit-exact vs the oracle.
#include "common.cuh"

namespace mf {

constexpr int kThreads = 256;
constexpr int kListCap = 512;            // keys scanned per round = 2 per thread
constexpr int kStage = 32;               // list entries whose values are staged in smem at once
constexpr int kVS = 1024;                // voxels per CTA segment: one float4 per thread and plane
constexpr int kSlots = 64;               // occupied voxels whose sums are resident per round
constexpr int kSlotsRound = kSlots - 3;  // a 4-voxel group never straddles two rounds
constexpr int kMaxCC = 48;               // channel planes per CTA

struct VoxGeom {
  float ox, oy, oz, pitch;
  int X, Y, Z, B;
};

// ---------------------------------------------------------------- prepass
// key[n] = b*V + flat voxel index, or -1 if out of bounds.  seg_start[b] / seg_end[b] are
// written by the points at the boundaries of b's run; entries of absent batches are never
// written, so the consumer validates what it reads against batch_indices instead of relying on
// an initialised workspace.  cta_flags[blockIdx.x] = OR of the MF_FLAG_* bits of this CTA's
// points (every slot is written: no memset).
__global__ void __launch_bounds__(kThreads)
k_avg_prepass(const float* __restrict__ points, const int* __restrict__ bi, long long N,
              VoxGeom g, int* __restrict__ keys, int* __restrict__ seg_start,
              int* __restrict__ seg_end, int* __restrict__ cta_flags) {
  const long long n = (long long)blockIdx.x * kThreads + threadIdx.x;
  int f = 0;
  if (n < N) {
    const float x = points[3 * n], y = points[3 * n + 1], z = points[3 * n + 2];
    const int b = bi[n];
    if (isnan(x) || isnan(y) || isnan(z)) f |= MF_FLAG_NAN_POINTS;
    const int ix = voxel_coord(x, g.ox, g.pitch);
    const int iy = voxel_coord(y, g.oy, g.pitch);
    const int iz = voxel_coord(z, g.oz, g.pitch);
    const bool okb = (b >= 0) && (b < g.B);
    if (!okb) f |= MF_FLAG_BAD_BATCH_INDEX;
    const bool ok = okb && ix >= 0 && ix < g.X && iy >= 0 && iy < g.Y && iz >= 0 && iz < g.Z;
    const int V = g.X * g.Y * g.Z;
    keys[n] = ok ? (b * V + (ix * g.Y + iy) * g.Z + iz) : -1;
    const int prev = (n > 0) ? bi[n - 1] : b;
    if (prev > b) f |= MF_FLAG_UNSORTED_BATCH;
    if (okb) {
      if (n == 0 || prev != b) seg_start[b] = (int)n;
      if (n == N - 1 || bi[n + 1] != b) seg_end[b] = (int)(n + 1);
    }
  }
  f = __reduce_or_sync(0xffffffffu, (unsigned)f);
  __shared__ int sf[kThreads / 32];
  if ((threadIdx.x & 31) == 0) sf[threadIdx.x >> 5] = f;
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) a |= sf[w];
    cta_flags[blockIdx.x] = a;
  }
}

// ---------------------------------------------------------------- forward
struct AvgParams {
  const float* values;
  const int* keys;
  const int* bi;
  const int* seg_start;
  const int* seg_end;
  const int* cta_flags;
  int n_key_ctas;
  long long N;
  int C, B, V;
  int CC;       // channels per chunk (grid.y chunks)
  int CCp;      // padded (odd) row length of the smem rows
  int LWs;      // log2 of the lane width LW >= CC of the staging / accumulate roles
  int segs_per_batch;
  int vec4;     // planes are 16-byte aligned and V % 4 == 0: float4 stores
  float* matrix;
  int* counts;
  int* flags_ws;     // workspace copy of the flag word (always written)
  int* flags_user;   // caller's flag word (OR-ed into), may be null
};

// A CTA owns (batch b, kVS = 1024 consecutive voxels, CC <= 48 channels).
//   gather  find the points of b that fall into its voxels (ordered compaction of the keys), sum
//           them per occupied voxel in ascending point order in shared memory, divide.  A handful
//           of dependent L2 round trips; every load batch is issued before its first use, and the
//           kernel is sized so that all CTAs are resident at once: the gathers of the whole grid
//           run while the memory system is still idle (the same loads take microseconds each
//           once 150 MB of stores are in flight).
//   stream  4 KiB of every channel plane of the chunk: one 16-byte store per thread and plane,
//           zeros straight from registers, occupied voxels patched in from shared memory.
// Every output element is written exactly once.
__global__ void __launch_bounds__(kThreads, 6)
k_avg_fused(AvgParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sums = reinterpret_cast<float*>(smem_raw);                 // [kSlots + 1][CCp], last = zeros
  float* stage = sums + (size_t)(kSlots + 1) * p.CCp;               // [kStage][CCp]
  int* list_n = reinterpret_cast<int*>(stage + (size_t)kStage * p.CCp);  // [kListCap] point id
  int* list_s = list_n + kListCap;                                  // [kListCap] slot
  int* cnt = list_s + kListCap;                                     // [kSlots + 1], last = 0
  int* base_s = cnt + kSlots + 1;                                   // [kThreads] first slot of a group
  unsigned* occ = reinterpret_cast<unsigned*>(base_s + kThreads);   // [kVS/32] occupancy bits
  __shared__ int s_warp[kThreads / 32];
  __shared__ int s_total, s_lo, s_hi;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x / p.segs_per_batch, seg = blockIdx.x - b * p.segs_per_batch;
  const int chunk = blockIdx.y;
  const int vbase = seg * kVS;
  const int vt = min(kVS, p.V - vbase);
  const int c0 = chunk * p.CC;
  const int cc = min(p.CC, p.C - c0);

  // ---- flag word of the call (per-CTA words of the prepass, OR-ed) and, in the same round
  // trip, the candidate run [seg_start, seg_end) of batch b with the entries that validate it
  int f = 0;
  for (int i = tid; i < p.n_key_ctas; i += kThreads) f |= __ldg(p.cta_flags + i);
  int cand_s = 0, cand_e = 0;
  bool okse = false;
  if (tid == 0 && p.N > 0) {
    const int s = p.seg_start[b], e = p.seg_end[b];
    const bool s_in = s >= 0 && s < p.N, e_in = e > 0 && e <= p.N;
    const int bs0 = s_in ? __ldg(p.bi + s) : -1, bs1 = (s_in && s > 0) ? __ldg(p.bi + s - 1) : -1;
    const int be0 = e_in ? __ldg(p.bi + e - 1) : -1, be1 = (e_in && e < p.N) ? __ldg(p.bi + e) : -1;
    okse = s_in && e_in && bs0 == b && (s == 0 || bs1 != b) && be0 == b && (e == p.N || be1 != b) && s < e;
    cand_s = s;
    cand_e = e;
  }
  const int unsorted = __syncthreads_or(f & MF_FLAG_UNSORTED_BATCH);
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    const int fn = __syncthreads_or(f & MF_FLAG_NAN_POINTS) ? MF_FLAG_NAN_POINTS : 0;
    const int fb = __syncthreads_or(f & MF_FLAG_BAD_BATCH_INDEX) ? MF_FLAG_BAD_BATCH_INDEX : 0;
    if (tid == 0) {
      const int all = fn | fb | (unsorted ? MF_FLAG_UNSORTED_BATCH : 0);
      *p.flags_ws = all;
      if (p.flags_user && all) atomicOr(p.flags_user, all);
    }
  }
  // the points of batch b: its run when batch_indices are sorted, else all points
  if (tid == 0) {
    long long lo = 0, hi = p.N;
    if (!unsorted) {
      lo = hi = 0;
      if (okse) { lo = cand_s; hi = cand_e; }
    }
    s_lo = (int)lo;
    s_hi = (int)hi;
  }
  for (int i = tid; i < kVS / 32; i += kThreads) occ[i] = 0u;
  for (int i = tid; i < p.CCp; i += kThreads) sums[kSlots * p.CCp + i] = 0.f;   // the zero row
  if (tid == 0) cnt[kSlots] = 0;
  __syncthreads();
  const int lo = s_lo, hi = s_hi;
  const int klo = b * p.V + vbase, khi = klo + vt;

  // ---- pass 1: occupancy bits of this segment
  for (int j = lo + tid; j < hi; j += kThreads) {
    const int k = __ldg(p.keys + j);
    if (k >= klo && k < khi) atomicOr(&occ[(k - klo) >> 5], 1u << ((k - klo) & 31));
  }
  __syncthreads();
  // thread t owns voxel group t (voxels 4t..4t+3): slots are numbered in voxel order
  const unsigned nib = (occ[tid >> 3] >> ((tid & 7) * 4)) & 0xFu;
  int my_base;
  {
    const int m = __popc(nib);
    int incl = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int woff = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) woff += (w < warp) ? s_warp[w] : 0;
    my_base = woff + incl - m;
    base_s[tid] = my_base;
    if (tid == kThreads - 1) s_total = woff + incl;
  }
  __syncthreads();
  const int n_occ = s_total;
  // trailing empty groups carry base == n_occ: they need a round of their own when n_occ is a
  // multiple of kSlotsRound
  const int n_rounds = n_occ / kSlotsRound + 1;
  const int my_round = my_base / kSlotsRound;
  // thread roles of the staging / accumulate / divide loops: NR rows x LW channel lanes
  const int LW = 1 << p.LWs, NR = kThreads >> p.LWs;
  const int g = tid >> p.LWs, c = tid & (LW - 1);
  const bool c_ok = c < cc;

  for (int r = 0; r < n_rounds; ++r) {
    const int n_used = min(kSlots, n_occ - r * kSlotsRound);   // slots this round can touch
    if (c_ok)
      for (int sl = g; sl < n_used; sl += NR) sums[sl * p.CCp + c] = 0.f;
    for (int e = tid; e < n_used; e += kThreads) cnt[e] = 0;
    __syncthreads();
    if (n_used > 0)
    for (int base = lo; base < hi; base += kListCap) {
      // ---- ordered compaction of the keys in [base, base+kListCap) that belong to round r
      const int i0 = base + 2 * tid;
      int sl[2];
      int m = 0;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        sl[j] = -1;
        if (i0 + j < hi) {
          const int k = __ldg(p.keys + i0 + j);
          if (k >= klo && k < khi) {
            const int v = k - klo, grp = v >> 2, bs = base_s[grp];
            if (bs / kSlotsRound == r) {
              const unsigned nb = (occ[grp >> 3] >> ((grp & 7) * 4)) & 0xFu;
              sl[j] = bs - r * kSlotsRound + __popc(nb & ((1u << (v & 3)) - 1u));
              ++m;
            }
          }
        }
      }
      int incl = m;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      if (lane == 31) s_warp[warp] = incl;
      __syncthreads();
      int woff = 0;
#pragma unroll
      for (int w = 0; w < kThreads / 32; ++w) woff += (w < warp) ? s_warp[w] : 0;
      if (tid == kThreads - 1) s_total = woff + incl;
      int pos = woff + incl - m;
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (sl[j] >= 0) {
          list_n[pos] = i0 + j;          // point id (N < 2^31 checked on host)
          list_s[pos] = sl[j];
          ++pos;
        }
      __syncthreads();
      const int L = s_total;
      // values of the listed points go through shared memory in batches of kStage rows; a thread
      // issues all its loads of a batch before the first store (independent L2 round trips)
      for (int l0 = 0; l0 < L; l0 += kStage) {
        const int nl = min(kStage, L - l0);
        if (c_ok) {
          float tmp[8];
          for (int lb = g; lb < nl; lb += 8 * NR) {
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int l = lb + u * NR;
              tmp[u] = l < nl ? __ldg(p.values + (long long)list_n[l0 + l] * p.C + c0 + c) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int l = lb + u * NR;
              if (l < nl) stage[l * p.CCp + c] = tmp[u];
            }
          }
        }
        __syncthreads();
        if (c_ok) {
          // row group g owns the slots s % NR == g: a slot's points are added in list order
          for (int l = 0; l < nl; ++l) {
            const int s = list_s[l0 + l];
            if ((s & (NR - 1)) == g) {
              sums[s * p.CCp + c] = __fadd_rn(sums[s * p.CCp + c], stage[l * p.CCp + c]);
              if (c == 0) cnt[s] += 1;
            }
          }
        }
        __syncthreads();
      }
    }
    // ---- averages in place
    if (c_ok)
      for (int sl = g; sl < n_used; sl += NR) {
        const int n = cnt[sl];
        if (n > 0) sums[sl * p.CCp + c] = __fdiv_rn(sums[sl * p.CCp + c], (float)n);
      }
    __syncthreads();
    // ---- stream this segment's piece of every plane of the chunk: groups of round r only.
    // One uniform loop: every lane reads its four voxels' values from shared memory -- empty
    // voxels point at an all-zero row -- so a warp never diverges and a plane costs four LDS,
    // one 16-byte store and no address arithmetic beyond the plane stride.
    if (my_round == r && 4 * tid < vt) {
      uint32_t a4[4];
      int c4[4];
      {
        int s = my_base - r * kSlotsRound;
        const uint32_t sb = static_cast<uint32_t>(__cvta_generic_to_shared(sums));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int slot = ((nib >> k) & 1u) ? s++ : kSlots;          // kSlots = the zero row
          a4[k] = sb + (uint32_t)(slot * p.CCp) * 4u;
          c4[k] = cnt[slot];
        }
      }
      const long long plane0 = ((long long)b * p.C + c0) * p.V + vbase + 4 * tid;
      if (p.vec4) {
        float4* d = reinterpret_cast<float4*>(p.matrix + plane0);
        const long long pstride = p.V >> 2;
#pragma unroll 8
        for (int ch = 0; ch < cc; ++ch, d += pstride) {
          float4 v;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v.x) : "r"(a4[0] + 4u * ch));
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v.y) : "r"(a4[1] + 4u * ch));
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v.z) : "r"(a4[2] + 4u * ch));
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v.w) : "r"(a4[3] + 4u * ch));
          __stcs(d, v);
        }
        if (chunk == 0)
          *reinterpret_cast<int4*>(p.counts + (long long)b * p.V + vbase + 4 * tid) =
              make_int4(c4[0], c4[1], c4[2], c4[3]);
      } else {
        // ragged / unaligned planes: scalar stores, tail guarded
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (4 * tid + k >= vt) break;
          float* dst = p.matrix + plane0 + k;
          for (int ch = 0; ch < cc; ++ch) {
            float v;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a4[k] + 4u * ch));
            dst[(long long)ch * p.V] = v;
          }
          if (chunk == 0) p.counts[(long long)b * p.V + vbase + 4 * tid + k] = c4[k];
        }
      }
    }
    __syncthreads();                                           // sums / cnt are reused by the next round
  }
}

// ---------------------------------------------------------------- backward
// gvalues[n,c] = gmatrix[b,c,idx] / counts[b,idx]   (average_voxelization_3d.py:170-206)
__global__ void k_avg_bwd(const float* __restrict__ gmatrix, const int* __restrict__ counts,
                          const float* __restrict__ points, const int* __restrict__ bi,
                          long long N, int C, VoxGeom g, float* __restrict__ gvalues) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  long long n = i / C;
  int c = (int)(i - n * C);
  int b = bi[n];
  int ix = voxel_coord(points[3 * n], g.ox, g.pitch);
  int iy = voxel_coord(points[3 * n + 1], g.oy, g.pitch);
  int iz = voxel_coord(points[3 * n + 2], g.oz, g.pitch);
  float out = 0.f;
  if (b >= 0 && b < g.B && ix >= 0 && ix < g.X && iy >= 0 && iy < g.Y && iz >= 0 && iz < g.Z) {
    long long V = (long long)g.X * g.Y * g.Z;
    long long flat = ((long long)ix * g.Y + iy) * g.Z + iz;
    out = __fdiv_rn(gmatrix[((long long)b * C + c) * V + flat], (float)counts[b * V + flat]);
  }
  gvalues[i] = out;
}

// ---------------------------------------------------------------- max voxelization
// order-preserving bits of a float.  -0 is folded onto +0 (-0 + 0 = +0 in round-to-nearest) so
// that the two compare equal, as `intensity > max_intensity` has them, and the lower point id
// wins.  The reference's result with a NaN intensity depends on arrival order (`>` is false both
// ways, so the first arrival keeps the voxel); here a NaN of either sign ranks above every number.
__device__ __forceinline__ unsigned int f2ord(float f) {
  if (f != f) return 0xffffffffu;
  unsigned int u = __float_as_uint(__fadd_rn(f, 0.f));
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// key = (orderable(intensity) << 32) | ~n : atomicMax -> max intensity, lowest n on ties
__global__ void k_max_scatter(const float* __restrict__ points, const int* __restrict__ bi,
                              const float* __restrict__ inten, long long N, VoxGeom g,
                              unsigned long long* __restrict__ keys, int* __restrict__ flags) {
  long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float x = points[3 * n], y = points[3 * n + 1], z = points[3 * n + 2];
  int b = bi[n];
  int f = 0;
  if (isnan(x) || isnan(y) || isnan(z)) f |= MF_FLAG_NAN_POINTS;
  int ix = voxel_coord(x, g.ox, g.pitch);
  int iy = voxel_coord(y, g.oy, g.pitch);
  int iz = voxel_coord(z, g.oz, g.pitch);
  bool okb = (b >= 0) && (b < g.B);
  if (!okb) f |= MF_FLAG_BAD_BATCH_INDEX;
  if (okb && ix >= 0 && ix < g.X && iy >= 0 && iy < g.Y && iz >= 0 && iz < g.Z) {
    long long V = (long long)g.X * g.Y * g.Z;
    long long flat = ((long long)ix * g.Y + iy) * g.Z + iz;
    unsigned long long key =
        ((unsigned long long)f2ord(inten[n]) << 32) | (unsigned long long)(~(unsigned int)n);
    atomicMax(&keys[b * V + flat], key);
  }
  if (f && flags) atomicOr(flags, f);
}

__global__ void k_max_gather(const float* __restrict__ values,
                             const unsigned long long* __restrict__ keys, int C, long long V,
                             long long BV, float* __restrict__ matrix, int* __restrict__ indices) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over B*C*V
  if (i >= BV * C) return;
  long long v = i % V;
  long long bc = i / V;
  int c = (int)(bc % C);
  long long b = bc / C;
  unsigned long long key = keys[b * V + v];
  int n = key ? (int)(~(unsigned int)(key & 0xffffffffu)) : -1;
  matrix[i] = (n >= 0) ? values[(long long)n * C + c] : 0.f;
  if (c == 0) indices[b * V + v] = n;
}

// gvalues[n,c] = gmatrix[b,c,v] for the (single) voxel n wins (max_voxelization_3d.py:158-179)
__global__ void k_max_bwd(const float* __restrict__ gmatrix, const int* __restrict__ indices,
                          int C, long long V, long long BV, float* __restrict__ gvalues) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BV * C) return;
  long long v = i % V;
  long long bc = i / V;
  int c = (int)(bc % C);
  long long b = bc / C;
  int n = indices[b * V + v];
  if (n >= 0) gvalues[(long long)n * C + c] = gmatrix[i];  // a point lies in exactly one voxel
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- store-pattern probe (diagnostics; scripts/fill_patterns.py).  All variants write the same
// B*(C+1)*V floats of zeros:
//   0  linear: CTA i streams 16 KiB contiguous (4 float4 per thread), st.cs
//   1  plane-strided: CTA = (1024 voxels, 48 planes), one float4 per thread and plane, st.cs
//   2  as 1 with default write-back stores
//   3  as 0 with default stores
//   4  plane-strided, CTA = (4096 voxels, 12 planes): 4 float4 per thread and plane, st.cs
__global__ void __launch_bounds__(256)
k_fill_probe(float* out, long long V, int planes, int mode) {
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (mode == 0 || mode == 3) {
    float4* dst = reinterpret_cast<float4*>(out) + (long long)blockIdx.x * 1024 + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (mode == 0) __stcs(dst + k * 256, z4); else dst[k * 256] = z4;
    }
    return;
  }
  if (mode == 4) {
    const int segs = (int)(V / 4096);
    const int seg = blockIdx.x % segs, b = blockIdx.x / segs;
    const int c0 = blockIdx.y * 12;
    float4* d = reinterpret_cast<float4*>(out + ((long long)b * planes + c0) * V + seg * 4096) + threadIdx.x;
    for (int ch = 0; ch < 12 && c0 + ch < planes; ++ch, d += V / 4)
#pragma unroll
      for (int k = 0; k < 4; ++k) __stcs(d + k * 256, z4);
    return;
  }
  const int segs = (int)(V / 1024);
  const int seg = blockIdx.x % segs, b = blockIdx.x / segs;
  const int c0 = blockIdx.y * 48;
  float4* d = reinterpret_cast<float4*>(out + ((long long)b * planes + c0) * V + seg * 1024) + threadIdx.x;
#pragma unroll 8
  for (int ch = 0; ch < 48 && c0 + ch < planes; ++ch, d += V / 4) {
    if (mode == 1) __stcs(d, z4); else *d = z4;
  }
}

}  // namespace mf

using namespace mf;

// workspace layout (nothing in it needs initialising):
//   [0]      int   flag word of the last call (mf_average_voxelization_3d_flags_offset)
//   [256]    int   seg_start[65536] | seg_end[65536]
//   [kWsCtaOff]    cta_flags[ceil(N/256)] | keys[N]
constexpr size_t kWsSegOff = 256;
constexpr size_t kWsCtaOff = kWsSegOff + 2 * 65536 * sizeof(int);

extern "C" int mf_debug_fill_probe(float* out, int B, int planes, int64_t V, int mode, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!out || B <= 0 || planes <= 0 || V % 4096 != 0 || mode < 0 || mode > 4) return MF_E_BADARG;
  const long long total = (long long)B * planes * V;
  if (mode == 0 || mode == 3) {
    k_fill_probe<<<(unsigned)(total / 4096), 256, 0, stream>>>(out, V, planes, mode);
  } else if (mode == 4) {
    dim3 g((unsigned)(B * (V / 4096)), (unsigned)((planes + 11) / 12));
    k_fill_probe<<<g, 256, 0, stream>>>(out, V, planes, mode);
  } else {
    dim3 g((unsigned)(B * (V / 1024)), (unsigned)((planes + 47) / 48));
    k_fill_probe<<<g, 256, 0, stream>>>(out, V, planes, mode);
  }
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" size_t mf_average_voxelization_3d_flags_offset(void) { return 0; }

static size_t avg_cta_bytes(int64_t n_points) {
  return align_up((size_t)((n_points > 0 ? n_points : 1) + 255) / 256 * 4, 256);
}

extern "C" size_t mf_average_voxelization_3d_workspace_bytes(int64_t n_points) {
  return kWsCtaOff + avg_cta_bytes(n_points) +
         align_up((size_t)(n_points > 0 ? n_points : 1) * 4, 256);
}

extern "C" int mf_average_voxelization_3d_fwd(
    const float* values, const float* points, const int32_t* batch_indices, int64_t N,
    int C, int B, float ox, float oy, float oz, float pitch, int X, int Y, int Z,
    float* matrix, int32_t* counts, void* workspace, size_t workspace_bytes, int32_t* flags,
    void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (N < 0 || C <= 0 || B <= 0 || X <= 0 || Y <= 0 || Z <= 0) return MF_E_BADARG;
  if (!matrix || !counts || !workspace) return MF_E_BADARG;
  if (N > 0 && (!values || !points || !batch_indices)) return MF_E_BADARG;
  long long V = (long long)X * Y * Z;
  if (V * B >= (1LL << 31) || N >= (1LL << 31)) return MF_E_TOOLARGE;
  if (B > 65535) return MF_E_TOOLARGE;
  if (workspace_bytes < mf_average_voxelization_3d_workspace_bytes(N)) return MF_E_WORKSPACE;

  char* ws = (char*)workspace;
  int* flags_ws = (int*)ws;
  int* seg_start = (int*)(ws + kWsSegOff);
  int* seg_end = seg_start + 65536;
  int* cta_flags = (int*)(ws + kWsCtaOff);
  int* keys = (int*)(ws + kWsCtaOff + avg_cta_bytes(N));
  VoxGeom g{ox, oy, oz, pitch, X, Y, Z, B};
  const int n_key_ctas = (int)div_up(N, kThreads);
  if (N > 0) {
    k_avg_prepass<<<n_key_ctas, kThreads, 0, stream>>>(points, batch_indices, N, g, keys,
                                                        seg_start, seg_end, cta_flags);
    MF_LAUNCH_CHECK();
  }
  AvgParams p;
  p.values = values; p.keys = keys; p.bi = batch_indices;
  p.seg_start = seg_start; p.seg_end = seg_end; p.cta_flags = cta_flags;
  p.n_key_ctas = N > 0 ? n_key_ctas : 0;
  p.N = N; p.C = C; p.B = B; p.V = (int)V;
  int nChunks = (C + kMaxCC - 1) / kMaxCC;
  p.CC = (C + nChunks - 1) / nChunks;
  nChunks = (C + p.CC - 1) / p.CC;
  p.CCp = p.CC | 1;
  p.LWs = 2;
  while ((1 << p.LWs) < p.CC) ++p.LWs;
  p.segs_per_batch = (int)((V + kVS - 1) / kVS);
  p.vec4 = (V % 4 == 0) && (((uintptr_t)matrix & 15) == 0) && (((uintptr_t)counts & 15) == 0);
  p.matrix = matrix; p.counts = counts;
  p.flags_ws = flags_ws; p.flags_user = flags;
  const long long n_cta = (long long)B * p.segs_per_batch;
  if (n_cta >= (1LL << 31) || nChunks > 65535) return MF_E_TOOLARGE;
  const size_t smem = (size_t)(kSlots + 1 + kStage) * p.CCp * 4 + (size_t)kListCap * 8 +
                      (size_t)(kSlots + 1) * 4 + (size_t)kThreads * 4 + (size_t)(kVS / 32) * 4;
  dim3 grid((unsigned)n_cta, (unsigned)nChunks, 1);
  k_avg_fused<<<grid, kThreads, smem, stream>>>(p);      // <= 25 KB of dynamic shared memory
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_average_voxelization_3d_bwd(
    const float* gmatrix, const int32_t* counts, const float* points,
    const int32_t* batch_indices, int64_t N, int C, int B, float ox, float oy, float oz,
    float pitch, int X, int Y, int Z, float* gvalues, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (N < 0 || C <= 0 || B <= 0 || X <= 0 || Y <= 0 || Z <= 0) return MF_E_BADARG;
  if (N == 0) return MF_OK;
  if (!gmatrix || !counts || !points || !batch_indices || !gvalues) return MF_E_BADARG;
  VoxGeom g{ox, oy, oz, pitch, X, Y, Z, B};
  k_avg_bwd<<<div_up(N * C, 256), 256, 0, stream>>>(gmatrix, counts, points, batch_indices, N, C,
                                                    g, gvalues);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" size_t mf_max_voxelization_3d_workspace_bytes(int B, int X, int Y, int Z) {
  return (size_t)B * X * Y * Z * 8;
}

extern "C" int mf_max_voxelization_3d_fwd(
    const float* values, const float* points, const int32_t* batch_indices,
    const float* intensities, int64_t N, int C, int B, float ox, float oy, float oz, float pitch,
    int X, int Y, int Z, float* matrix, int32_t* indices, void* workspace,
    size_t workspace_bytes, int32_t* flags, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (N < 0 || C <= 0 || B <= 0 || X <= 0 || Y <= 0 || Z <= 0) return MF_E_BADARG;
  if (!matrix || !indices || !workspace) return MF_E_BADARG;
  if (N > 0 && (!values || !points || !batch_indices || !intensities)) return MF_E_BADARG;
  if (N >= (1LL << 31)) return MF_E_TOOLARGE;
  long long V = (long long)X * Y * Z, BV = V * B;
  if (workspace_bytes < (size_t)BV * 8) return MF_E_WORKSPACE;
  unsigned long long* keys = (unsigned long long*)workspace;
  MF_CUDA_TRY(cudaMemsetAsync(keys, 0, (size_t)BV * 8, stream));
  VoxGeom g{ox, oy, oz, pitch, X, Y, Z, B};
  if (N > 0) {
    k_max_scatter<<<div_up(N, 256), 256, 0, stream>>>(points, batch_indices, intensities, N, g,
                                                      keys, flags);
    MF_LAUNCH_CHECK();
  }
  k_max_gather<<<div_up(BV * C, 256), 256, 0, stream>>>(values, keys, C, V, BV, matrix, indices);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_max_voxelization_3d_bwd(const float* gmatrix, const int32_t* indices, int64_t N,
                                          int C, int B, int X, int Y, int Z, float* gvalues,
                                          void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (N < 0 || C <= 0 || B <= 0 || X <= 0 || Y <= 0 || Z <= 0) return MF_E_BADARG;
  if (N == 0) return MF_OK;
  if (!gmatrix || !indices || !gvalues) return MF_E_BADARG;
  long long V = (long long)X * Y * Z, BV = V * B;
  MF_CUDA_TRY(cudaMemsetAsync(gvalues, 0, (size_t)N * C * 4, stream));
  k_max_bwd<<<div_up(BV * C, 256), 256, 0, stream>>>(gmatrix, indices, C, V, BV, gvalues);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
