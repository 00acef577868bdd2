// Point-to-point ICP of contrib.ICPRegistration (morefusion/contrib/icp_registration.py), the
// Open3D calls it makes restated in float64 (oracle/icp.py): voxel down-sampling, a uniform cell
// list over the CAD cloud, and every iteration of every instance in one launch.
//
// Built with -fmad=false: the voxel keys, the down-sampled means and the d^2 threshold tests are
// the oracle's float64 expressions, rounded step by step.  With g++ -DMF_HOST_EMU (and
// -ffp-contract=off) only the per-thread helpers compile: cell_window, nearest, horn_rotation and
// apply, which tests/emu/icp_emu.cpp runs on the host.
#include <float.h>
#include <limits.h>
#include <math.h>

#ifdef MF_HOST_EMU
#include "mapping_emu_stubs.h"
#include "../../include/morefusion_b200.h"
#else
#include "common.cuh"
#endif

namespace {

constexpr int SORT_THREADS = 512;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int RUN_THREADS = 256;
constexpr int RUN_WARPS = RUN_THREADS / 32;
constexpr int RUN_SMEM_POINTS = 4096;       // source points kept in shared memory up to this many

template <typename T>
__device__ __forceinline__ double ld(const T* p, long long i) { return (double)p[i]; }

// floor((x - origin) / size) clamped to [0, INT_MAX]: a key below 0 cannot occur for a point of
// the cloud itself.  A point's key is INT_MAX only when it does not fit (KEY_MAX below): the
// cloud is then refused rather than having distinct voxels merged at the clamp.
__device__ __forceinline__ int cell_of(double x, double origin, double size) {
  double c = floor((x - origin) / size);
  if (!(c > 0.0)) return 0;
  if (c >= (double)INT_MAX) return INT_MAX;
  return (int)c;
}

constexpr int KEY_MAX = INT_MAX - 1;        // the largest key a sorted cloud holds

// The cells [*lo, *hi] on one axis that can hold a point within r of x: those of x - r and x + r,
// both capped at KEY_MAX.  No key of a cell list exceeds KEY_MAX, so the cap drops no candidate,
// and a loop `for (c = lo; c <= hi; ++c)` ends: with hi = INT_MAX, ++c would overflow instead
// (a query at origin + (2^31 - 1) h or beyond, e.g. an init 1e8 m off at h = 2 cm).
__device__ __forceinline__ void cell_window(double x, double r, double origin, double h, int* lo,
                                            int* hi) {
  *lo = min(cell_of(x - r, origin, h), KEY_MAX);
  *hi = min(cell_of(x + r, origin, h), KEY_MAX);
}

#ifndef MF_HOST_EMU

__device__ __forceinline__ int axis(int4 v, int a) { return a == 0 ? v.x : (a == 1 ? v.y : v.z); }

// exclusive prefix count of `flag` over the block; *total gets the block's count
template <int WARPS>
__device__ int block_scan_flag(bool flag, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) s_warp[w] = __popc(b);
  __syncthreads();
  if (w == 0) {
    const int v = lane < WARPS ? s_warp[lane] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane < WARPS) s_warp[lane] = x - v;
    if (lane == 31) s_warp[32] = x;
  }
  __syncthreads();
  const int r = s_warp[w] + __popc(b & ((1u << lane) - 1u));
  *total = s_warp[32];
  __syncthreads();
  return r;
}

// One CTA per cloud m.  Rows [0, n_rows) of points[m] whose three coordinates are finite get the
// key floor((p - min_bound) / size), min_bound = min(p) - size / 2 (float64), and are sorted
// stably by (i, j, k): an LSD radix sort over the bytes the keys use, k's first.
//   down-sampling (CELLS = false): one output row per occupied voxel, in ascending (i, j, k):
//     the float64 mean of its points summed in ascending row order, its key and its count
//     (out_aux); n_out[m] = the number of voxels.
//   cell list (CELLS = true): every point in key order with its key and its row (out_aux);
//     out_origin[m] = min_bound.
template <typename T, bool CELLS>
__global__ void __launch_bounds__(SORT_THREADS)
k_icp_sort(const T* __restrict__ points, int N, const int32_t* __restrict__ n_rows_dev, double size,
           int4* __restrict__ buf_a, int4* __restrict__ buf_b, double* __restrict__ out_points,
           int32_t* __restrict__ out_keys, int32_t* __restrict__ out_aux,
           int32_t* __restrict__ n_out, double* __restrict__ out_origin) {
  __shared__ int s_hist[SORT_WARPS][256];
  __shared__ int s_tot[256];
  __shared__ int s_warp[33];
  __shared__ double s_red[SORT_WARPS][3];
  __shared__ int s_ired[SORT_WARPS][3];
  const int m = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const long long base = (long long)m * N;
  const T* P = points + base * 3;
  int4* A = buf_a + base;
  int4* B = buf_b + base;
  const int n_rows = n_rows_dev ? min(max(n_rows_dev[m], 0), N) : N;

  // min over the finite rows
  double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX};
  for (int r = tid; r < n_rows; r += SORT_THREADS) {
    const double x = ld(P, 3ll * r), y = ld(P, 3ll * r + 1), z = ld(P, 3ll * r + 2);
    if (isfinite(x) && isfinite(y) && isfinite(z)) {
      mn[0] = fmin(mn[0], x); mn[1] = fmin(mn[1], y); mn[2] = fmin(mn[2], z);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn[a] = fmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
    if (lane == 0) s_red[w][a] = mn[a];
  }
  __syncthreads();
  double mb[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double v = DBL_MAX;
    for (int i = 0; i < SORT_WARPS; ++i) v = fmin(v, s_red[i][a]);
    mb[a] = v - 0.5 * size;
  }

  // the finite rows in row order, with their keys
  int n = 0, kmax[3] = {0, 0, 0};
  for (int r0 = 0; r0 < n_rows; r0 += SORT_THREADS) {
    const int r = r0 + tid;
    double x = 0, y = 0, z = 0;
    bool ok = false;
    if (r < n_rows) {
      x = ld(P, 3ll * r); y = ld(P, 3ll * r + 1); z = ld(P, 3ll * r + 2);
      ok = isfinite(x) && isfinite(y) && isfinite(z);
    }
    int total;
    const int at = n + block_scan_flag<SORT_WARPS>(ok, s_warp, &total);
    if (ok) {
      const int4 k = make_int4(cell_of(x, mb[0], size), cell_of(y, mb[1], size),
                               cell_of(z, mb[2], size), r);
      kmax[0] = max(kmax[0], k.x); kmax[1] = max(kmax[1], k.y); kmax[2] = max(kmax[2], k.z);
      A[at] = k;
    }
    n += total;
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kmax[a] = max(kmax[a], __shfl_xor_sync(0xffffffffu, kmax[a], o));
    if (lane == 0) s_ired[w][a] = kmax[a];
  }
  __syncthreads();
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    int v = 0;
    for (int i = 0; i < SORT_WARPS; ++i) v = max(v, s_ired[i][a]);
    kmax[a] = v;
  }
  // a key past KEY_MAX does not fit in int32: refuse the cloud (n_out = -1, or a NaN origin)
  // rather than merge the voxels beyond it; k_icp_run refuses such a source or target in turn
  if (kmax[0] > KEY_MAX || kmax[1] > KEY_MAX || kmax[2] > KEY_MAX) {
    if (CELLS && tid < 3) out_origin[3 * m + tid] = nan("");
    if (!CELLS && tid == 0) n_out[m] = -1;
    return;
  }

  // each warp owns a contiguous chunk, so a digit's items keep their order: the sort is stable
  const int chunk = (n + SORT_WARPS - 1) / SORT_WARPS;
  const int lo = min(n, w * chunk), hi = min(n, lo + chunk);
  int4 *src = A, *dst = B;
  for (int a = 2; a >= 0; --a) {
    for (int shift = 0; shift < 32 && (kmax[a] >> shift) != 0; shift += 8) {
      for (int i = tid; i < SORT_WARPS * 256; i += SORT_THREADS) (&s_hist[0][0])[i] = 0;
      __syncthreads();
      for (int b0 = lo; b0 < hi; b0 += 32) {
        const int i = b0 + lane;
        const unsigned am = __ballot_sync(0xffffffffu, i < hi);
        if (i < hi) {
          const int d = (axis(src[i], a) >> shift) & 255;
          const unsigned peers = __match_any_sync(am, d);
          if (lane == __ffs(peers) - 1) s_hist[w][d] += __popc(peers);
        }
        __syncwarp();
      }
      __syncthreads();
      if (tid < 256) {
        int t = 0;
        for (int i = 0; i < SORT_WARPS; ++i) t += s_hist[i][tid];
        s_tot[tid] = t;
      }
      __syncthreads();
      if (tid == 0) {
        int run = 0;
        for (int d = 0; d < 256; ++d) {
          const int t = s_tot[d];
          s_tot[d] = run;
          run += t;
        }
      }
      __syncthreads();
      if (tid < 256) {
        int run = s_tot[tid];
        for (int i = 0; i < SORT_WARPS; ++i) {
          const int t = s_hist[i][tid];
          s_hist[i][tid] = run;
          run += t;
        }
      }
      __syncthreads();
      for (int b0 = lo; b0 < hi; b0 += 32) {
        const int i = b0 + lane;
        const unsigned am = __ballot_sync(0xffffffffu, i < hi);
        int d = 0, pos = 0, cnt = 0;
        bool lead = false;
        int4 v;
        if (i < hi) {
          v = src[i];
          d = (axis(v, a) >> shift) & 255;
          const unsigned peers = __match_any_sync(am, d);
          pos = s_hist[w][d] + __popc(peers & ((1u << lane) - 1u));
          lead = lane == __ffs(peers) - 1;
          cnt = __popc(peers);
          dst[pos] = v;
        }
        __syncwarp();
        if (lead) s_hist[w][d] += cnt;
        __syncwarp();
      }
      __syncthreads();
      int4* t = src;
      src = dst;
      dst = t;
    }
  }

  if (CELLS) {
    for (int i = tid; i < n; i += SORT_THREADS) {
      const int4 k = src[i];
      const long long o = base + i;
      out_points[3 * o] = ld(P, 3ll * k.w);
      out_points[3 * o + 1] = ld(P, 3ll * k.w + 1);
      out_points[3 * o + 2] = ld(P, 3ll * k.w + 2);
      out_keys[3 * o] = k.x; out_keys[3 * o + 1] = k.y; out_keys[3 * o + 2] = k.z;
      out_aux[o] = k.w;
    }
    if (tid < 3) out_origin[3 * m + tid] = mb[tid];
    return;
  }
  // segment heads -> the voxel starts (written into the free buffer), then one thread per voxel
  int* starts = reinterpret_cast<int*>(dst);
  int nv = 0;
  for (int i0 = 0; i0 < n; i0 += SORT_THREADS) {
    const int i = i0 + tid;
    bool head = false;
    if (i < n) {
      const int4 k = src[i];
      head = i == 0;
      if (!head) {
        const int4 p = src[i - 1];
        head = p.x != k.x || p.y != k.y || p.z != k.z;
      }
    }
    int total;
    const int at = nv + block_scan_flag<SORT_WARPS>(head, s_warp, &total);
    if (head) starts[at] = i;
    nv += total;
  }
  __syncthreads();
  for (int v = tid; v < nv; v += SORT_THREADS) {
    const int s = starts[v], e = v + 1 < nv ? starts[v + 1] : n;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int i = s; i < e; ++i) {
      const int r = src[i].w;
      sx = sx + ld(P, 3ll * r);
      sy = sy + ld(P, 3ll * r + 1);
      sz = sz + ld(P, 3ll * r + 2);
    }
    const double c = (double)(e - s);
    const int4 k = src[s];
    const long long o = base + v;
    out_points[3 * o] = sx / c;
    out_points[3 * o + 1] = sy / c;
    out_points[3 * o + 2] = sz / c;
    out_keys[3 * o] = k.x; out_keys[3 * o + 1] = k.y; out_keys[3 * o + 2] = k.z;
    out_aux[o] = e - s;
  }
  if (tid == 0) n_out[m] = nv;
}

// ----------------------------------------------------------------------------------------- ICP

// sum of K doubles over the block in a fixed order (xor butterfly per warp, then the warps in
// order); every thread gets the sums
template <int K>
__device__ void block_sum(double* v, double (*s)[K], double* s_out) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = v[k] + __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) s[w][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double t = 0.0;
    for (int i = 0; i < RUN_WARPS; ++i) t = t + s[i][threadIdx.x];
    s_out[threadIdx.x] = t;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = s_out[k];
  __syncthreads();
}

#endif  // !MF_HOST_EMU

__device__ __forceinline__ void apply(const double* T, double& x, double& y, double& z) {
  const double a = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
  const double b = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
  const double c = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
  x = a; y = b; z = c;
}

// the nearest target point of q (lowest index among equals) with d^2 < r2, else -1.  Every target
// with computed d^2 < r2 has |q_a - t_a| < r on each axis, so fl(q_a - r) <= t_a <= fl(q_a + r)
// and, floor((x - o) / h) being monotone in x, its cell lies in the window scanned here: the
// search over the cell list is exact.
__device__ int nearest(double qx, double qy, double qz, const mf_icp_target& tg, int nt, double r,
                       double r2, double* d2_out) {
  const double h = tg.cell_size;
  int i0, i1, j0, j1, k0, k1;
  cell_window(qx, r, tg.origin[0], h, &i0, &i1);
  cell_window(qy, r, tg.origin[1], h, &j0, &j1);
  cell_window(qz, r, tg.origin[2], h, &k0, &k1);
  const int* C = tg.cells;
  double best = r2;
  int bi = -1, bidx = INT_MAX;
  for (int ci = i0; ci <= i1; ++ci) {
    for (int cj = j0; cj <= j1; ++cj) {
      // first entry >= (ci, cj, k0)
      int l = 0, u = nt;
      while (l < u) {
        const int mid = (l + u) >> 1;
        const int a = C[3 * mid], b = C[3 * mid + 1], c = C[3 * mid + 2];
        const bool less = a != ci ? a < ci : (b != cj ? b < cj : c < k0);
        if (less) l = mid + 1; else u = mid;
      }
      for (int t = l; t < nt; ++t) {
        if (C[3 * t] != ci || C[3 * t + 1] != cj || C[3 * t + 2] > k1) break;
        const double dx = qx - tg.points[3 * t], dy = qy - tg.points[3 * t + 1],
                     dz = qz - tg.points[3 * t + 2];
        const double d2 = (dx * dx + dy * dy) + dz * dz;
        const int idx = tg.index[t];
        if (d2 < best || (d2 == best && bi >= 0 && idx < bidx)) {
          best = d2;
          bi = t;
          bidx = idx;
        }
      }
    }
  }
  *d2_out = best;
  return bi;
}

// Horn's closed form of the Umeyama rotation: the unit eigenvector of the largest eigenvalue of
// the symmetric 4x4 N(S), S[a][b] = sum (s_a - s_mean_a)(t_b - t_mean_b), is the quaternion
// (w, x, y, z) of the R in SO(3) that maximises tr(R^T sigma) -- the R = U diag(1, 1, det) V^T of
// the SVD route wherever that optimum is unique.  Cyclic Jacobi; equal eigenvalues go to the
// lowest index, so S = 0 (one correspondence) gives R = I.
__device__ void horn_rotation(const double* C, double* R) {
  // C[3 i + j] = sum (t_i - tm_i)(s_j - sm_j), so S[a][b] = C[3 b + a]
  const double Sxx = C[0], Syx = C[1], Szx = C[2];
  const double Sxy = C[3], Syy = C[4], Szy = C[5];
  const double Sxz = C[6], Syz = C[7], Szz = C[8];
  double A[4][4] = {{Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx},
                    {Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz},
                    {Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy},
                    {Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz}};
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) off += fabs(A[p][q]);
    if (off == 0.0) break;
    for (int p = 0; p < 3; ++p) {
      for (int q = p + 1; q < 4; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double g = 100.0 * fabs(apq);
        if (sweep > 3 && fabs(A[p][p]) + g == fabs(A[p][p]) && fabs(A[q][q]) + g == fabs(A[q][q])) {
          A[p][q] = A[q][p] = 0.0;
          continue;
        }
        const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
        double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
        if (theta < 0.0) t = -t;
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 4; ++k) {           // A <- A J (columns p, q)
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 4; ++k) {           // A <- J^T A (rows p, q)
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        A[p][q] = A[q][p] = 0.0;
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
    }
  }
  int b = 0;
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > A[b][b]) b = k;
  double w = V[0][b], x = V[1][b], y = V[2][b], z = V[3][b];
  const double nq = sqrt(((w * w + x * x) + y * y) + z * z);
  w /= nq; x /= nq; y /= nq; z /= nq;
  R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - w * z); R[2] = 2.0 * (x * z + w * y);
  R[3] = 2.0 * (x * y + w * z); R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - w * x);
  R[6] = 2.0 * (x * z - w * y); R[7] = 2.0 * (y * z + w * x); R[8] = 1.0 - 2.0 * (x * x + y * y);
}

#ifndef MF_HOST_EMU

// One CTA per instance: Open3D's RegistrationICP loop (oracle/icp.py) from init to convergence
// or max_iteration, the source points resident in shared memory when they fit (else in `work`).
__global__ void __launch_bounds__(RUN_THREADS)
k_icp_run(const double* __restrict__ source, int N, const int32_t* __restrict__ n_source,
          const mf_icp_target* __restrict__ targets, const double* __restrict__ init, double r,
          int max_iteration, double rel_fitness, double rel_rmse, int smem_points,
          double* __restrict__ work, int32_t* __restrict__ match_ws, double* __restrict__ out_T,
          double* __restrict__ out_fitness, double* __restrict__ out_rmse,
          int32_t* __restrict__ out_iterations) {
  extern __shared__ double s_pts[];
  __shared__ double s_red[RUN_WARPS][9];
  __shared__ double s_sum[9];
  __shared__ double s_T[16], s_U[16];
  const int m = blockIdx.x, tid = threadIdx.x;
  const int n = max(0, min(n_source[m], N));
  const long long base = (long long)m * N;
  double* Pp = n <= smem_points ? s_pts : work + 3 * base;
  int32_t* match = match_ws + base;
  const mf_icp_target tg = targets[m];
  const int nt = *tg.count;
  const double r2 = r * r;
  // a source or target cloud k_icp_sort refused (a key past KEY_MAX): NaN out, no iteration
  if (n_source[m] < 0 || nt < 0 ||
      !(isfinite(tg.origin[0]) && isfinite(tg.origin[1]) && isfinite(tg.origin[2]))) {
    if (tid < 16) out_T[16 * m + tid] = nan("");
    if (tid == 0) {
      out_fitness[m] = nan("");
      out_rmse[m] = nan("");
      out_iterations[m] = 0;
    }
    return;
  }
  if (tid < 16) s_T[tid] = init[16 * m + tid];
  __syncthreads();
  for (int i = tid; i < n; i += RUN_THREADS) {
    double x = source[3 * (base + i)], y = source[3 * (base + i) + 1], z = source[3 * (base + i) + 2];
    apply(s_T, x, y, z);
    Pp[3 * i] = x; Pp[3 * i + 1] = y; Pp[3 * i + 2] = z;
  }
  __syncthreads();

  // correspondences: count, sum d^2, sum of matched source and target points
  auto correspond = [&](double* acc) {
    for (int k = 0; k < 8; ++k) acc[k] = 0.0;
    for (int i = tid; i < n; i += RUN_THREADS) {
      const double x = Pp[3 * i], y = Pp[3 * i + 1], z = Pp[3 * i + 2];
      double d2;
      const int t = nt > 0 ? nearest(x, y, z, tg, nt, r, r2, &d2) : -1;
      match[i] = t;
      if (t >= 0) {
        acc[0] = acc[0] + 1.0;
        acc[1] = acc[1] + d2;
        acc[2] = acc[2] + x; acc[3] = acc[3] + y; acc[4] = acc[4] + z;
        acc[5] = acc[5] + tg.points[3 * t]; acc[6] = acc[6] + tg.points[3 * t + 1];
        acc[7] = acc[7] + tg.points[3 * t + 2];
      }
    }
    block_sum<8>(acc, reinterpret_cast<double(*)[8]>(&s_red[0][0]), s_sum);
  };
  auto fit_rmse = [&](const double* acc, double& f, double& e) {
    if (acc[0] == 0.0) { f = 0.0; e = 0.0; return; }
    f = acc[0] / (double)n;
    e = sqrt(acc[1] / acc[0]);
  };

  double acc[9];
  correspond(acc);
  double fit, rmse;
  fit_rmse(acc, fit, rmse);
  int it = 0;
  for (it = 1; it <= max_iteration; ++it) {
    const double cnt = acc[0];
    double sm[3] = {0, 0, 0}, tm[3] = {0, 0, 0};
    if (cnt > 0.0) {
      for (int a = 0; a < 3; ++a) { sm[a] = acc[2 + a] / cnt; tm[a] = acc[5 + a] / cnt; }
    }
    double cov[9];
    for (int k = 0; k < 9; ++k) cov[k] = 0.0;
    for (int i = tid; i < n; i += RUN_THREADS) {
      const int t = match[i];
      if (t < 0) continue;
      const double s[3] = {Pp[3 * i] - sm[0], Pp[3 * i + 1] - sm[1], Pp[3 * i + 2] - sm[2]};
      const double d[3] = {tg.points[3 * t] - tm[0], tg.points[3 * t + 1] - tm[1],
                           tg.points[3 * t + 2] - tm[2]};
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) cov[3 * a + b] = cov[3 * a + b] + d[a] * s[b];
    }
    block_sum<9>(cov, s_red, s_sum);
    if (tid == 0) {
      double U[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
      if (cnt > 0.0) {
        double R[9];
        horn_rotation(cov, R);
        for (int a = 0; a < 3; ++a) {
          for (int b = 0; b < 3; ++b) U[4 * a + b] = R[3 * a + b];
          U[4 * a + 3] = tm[a] - ((R[3 * a] * sm[0] + R[3 * a + 1] * sm[1]) + R[3 * a + 2] * sm[2]);
        }
      }
      double T[16];
      for (int a = 0; a < 4; ++a)
        for (int b = 0; b < 4; ++b)
          T[4 * a + b] = ((U[4 * a] * s_T[b] + U[4 * a + 1] * s_T[4 + b]) + U[4 * a + 2] * s_T[8 + b]) +
                         U[4 * a + 3] * s_T[12 + b];
      for (int k = 0; k < 16; ++k) { s_T[k] = T[k]; s_U[k] = U[k]; }
    }
    __syncthreads();
    for (int i = tid; i < n; i += RUN_THREADS) {
      double x = Pp[3 * i], y = Pp[3 * i + 1], z = Pp[3 * i + 2];
      apply(s_U, x, y, z);
      Pp[3 * i] = x; Pp[3 * i + 1] = y; Pp[3 * i + 2] = z;
    }
    __syncthreads();
    const double fit0 = fit, rmse0 = rmse;
    correspond(acc);
    fit_rmse(acc, fit, rmse);
    if (fabs(fit0 - fit) < rel_fitness && fabs(rmse0 - rmse) < rel_rmse) break;
  }
  if (it > max_iteration) it = max_iteration;
  if (tid < 16) out_T[16 * m + tid] = s_T[tid];
  if (tid == 0) {
    out_fitness[m] = fit;
    out_rmse[m] = rmse;
    out_iterations[m] = it;
  }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

#endif  // !MF_HOST_EMU

}  // namespace

#ifndef MF_HOST_EMU
extern "C" size_t mf_icp_sort_workspace_bytes(int M, int N) {
  if (M < 0 || N < 0) return 0;
  return 2 * align256((size_t)M * N * sizeof(int4));
}

extern "C" int mf_icp_voxel_down_sample(const void* points, int points_f64, int M, int N,
                                        double voxel_size, double* means, int32_t* keys,
                                        int32_t* counts, int32_t* n_out, void* workspace,
                                        size_t workspace_bytes, void* stream_) {
  if (M < 0 || N < 1 || !(voxel_size > 0.0) || !isfinite(voxel_size)) return MF_E_BADARG;
  if (M == 0) return MF_OK;
  if (!points || !means || !keys || !counts || !n_out || !workspace) return MF_E_BADARG;
  if ((long long)M * N > INT_MAX) return MF_E_TOOLARGE;
  if (workspace_bytes < mf_icp_sort_workspace_bytes(M, N)) return MF_E_WORKSPACE;
  int4* a = (int4*)workspace;
  int4* b = (int4*)((char*)workspace + align256((size_t)M * N * sizeof(int4)));
  cudaStream_t st = (cudaStream_t)stream_;
  if (points_f64) {
    MF_PREFER_MAX_SMEM((k_icp_sort<double, false>));
    k_icp_sort<double, false><<<M, SORT_THREADS, 0, st>>>(
        (const double*)points, N, nullptr, voxel_size, a, b, means, keys, counts, n_out, nullptr);
  } else {
    MF_PREFER_MAX_SMEM((k_icp_sort<float, false>));
    k_icp_sort<float, false><<<M, SORT_THREADS, 0, st>>>(
        (const float*)points, N, nullptr, voxel_size, a, b, means, keys, counts, n_out, nullptr);
  }
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" int mf_icp_cell_list(const double* points, const int32_t* n_points, int N,
                                double cell_size, double* sorted_points, int32_t* cells,
                                int32_t* index, double* origin, void* workspace,
                                size_t workspace_bytes, void* stream_) {
  if (N < 1 || !(cell_size > 0.0) || !isfinite(cell_size) || !points || !n_points ||
      !sorted_points || !cells || !index || !origin || !workspace)
    return MF_E_BADARG;
  if (workspace_bytes < mf_icp_sort_workspace_bytes(1, N)) return MF_E_WORKSPACE;
  int4* a = (int4*)workspace;
  int4* b = (int4*)((char*)workspace + align256((size_t)N * sizeof(int4)));
  MF_PREFER_MAX_SMEM((k_icp_sort<double, true>));
  k_icp_sort<double, true><<<1, SORT_THREADS, 0, (cudaStream_t)stream_>>>(
      points, N, n_points, cell_size, a, b, sorted_points, cells, index, nullptr, origin);
  MF_LAUNCH_CHECK();
  return MF_OK;
}

extern "C" size_t mf_icp_run_workspace_bytes(int M, int N) {
  if (M < 0 || N < 0) return 0;
  return align256((size_t)M * N * 3 * sizeof(double)) + align256((size_t)M * N * sizeof(int32_t));
}

extern "C" int mf_icp_run(int M, const double* source, int N, const int32_t* n_source,
                          const mf_icp_target* targets, const double* transform_init,
                          const double* transform_init_host,
                          double max_distance, int max_iteration, double relative_fitness,
                          double relative_rmse, double* transform, double* fitness, double* rmse,
                          int32_t* iterations, void* workspace, size_t workspace_bytes,
                          void* stream_) {
  if (M < 0 || N < 1 || max_iteration < 0 || !(max_distance > 0.0) || !isfinite(max_distance) ||
      !(relative_fitness >= 0.0) || !(relative_rmse >= 0.0))
    return MF_E_BADARG;
  if (M == 0) return MF_OK;
  if (!source || !n_source || !targets || !transform_init || !transform_init_host || !transform ||
      !fitness ||
      !rmse || !iterations || !workspace)
    return MF_E_BADARG;
  for (long long i = 0; i < 16ll * M; ++i)
    if (!isfinite(transform_init_host[i])) return MF_E_BADARG;
  if ((long long)M * N > INT_MAX) return MF_E_TOOLARGE;
  if (workspace_bytes < mf_icp_run_workspace_bytes(M, N)) return MF_E_WORKSPACE;
  char* w = (char*)workspace;
  double* pts = (double*)w;
  w += align256((size_t)M * N * 3 * sizeof(double));
  int32_t* match = (int32_t*)w;
  cudaStream_t st = (cudaStream_t)stream_;
  const int smem_points = N < RUN_SMEM_POINTS ? N : RUN_SMEM_POINTS;
  const size_t smem = (size_t)smem_points * 3 * sizeof(double);
  MF_ENSURE_DYN_SMEM(k_icp_run, smem);
  k_icp_run<<<M, RUN_THREADS, smem, st>>>(source, N, n_source, targets, transform_init,
                                          max_distance,
                                          max_iteration, relative_fitness, relative_rmse,
                                          smem_points, pts, match, transform, fitness, rmse,
                                          iterations);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
#endif  // !MF_HOST_EMU
