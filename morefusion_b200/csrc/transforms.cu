// Rigid-transform operators (sm_90a).
//
// Replaces (morefusion/functions/geometry):
//   quaternion_matrix.py:6-78  (q*sqrt(2/|q|^2), outer product, 9-entry table + its backward)
//   compose_transform.py:5-48, translation_matrix.py:5-39, transformation_matrix.py:5-18
//   transform_points.py:6-30   ((M,4,4)@(4,P) via F.matmul -> one fused kernel)
#include "common.cuh"

namespace mf {

__device__ __forceinline__ void quat_to_rot(const float q[4], float R[9]) {
  float n = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[1], q[1])),
                                __fmul_rn(q[2], q[2])), __fmul_rn(q[3], q[3]));
  float s = __fsqrt_rn(__fdiv_rn(2.f, n));
  float w = __fmul_rn(q[0], s), x = __fmul_rn(q[1], s), y = __fmul_rn(q[2], s),
        z = __fmul_rn(q[3], s);
  float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
  float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
  float xw = __fmul_rn(x, w), yw = __fmul_rn(y, w), zw = __fmul_rn(z, w);
  R[0] = __fsub_rn(__fsub_rn(1.f, yy), zz);
  R[1] = __fsub_rn(xy, zw);
  R[2] = __fadd_rn(xz, yw);
  R[3] = __fadd_rn(xy, zw);
  R[4] = __fsub_rn(__fsub_rn(1.f, xx), zz);
  R[5] = __fsub_rn(yz, xw);
  R[6] = __fsub_rn(xz, yw);
  R[7] = __fadd_rn(yz, xw);
  R[8] = __fsub_rn(__fsub_rn(1.f, xx), yy);
}

// gR (3x3 block, row-major 9) -> gq, through table(:41-49) -> outer -> scale
__device__ __forceinline__ void quat_bwd(const float q[4], const float gR[9], float gq[4]) {
  float n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  float s = sqrtf(2.f / n);
  float qs[4] = {q[0] * s, q[1] * s, q[2] * s, q[3] * s};
  // gQ[a][b] non-zero entries (indices 0..3 = w,x,y,z)
  float g10 = -gR[5] + gR[7];
  float g11 = -gR[4] - gR[8];
  float g12 = gR[1] + gR[3];
  float g13 = gR[2] + gR[6];
  float g20 = gR[2] - gR[6];
  float g22 = -gR[0] - gR[8];
  float g23 = gR[5] + gR[7];
  float g30 = -gR[1] + gR[3];
  float g33 = -gR[0] - gR[4];
  // gqs = gQ qs + gQ^T qs
  float gqs[4];
  gqs[0] = g10 * qs[1] + g20 * qs[2] + g30 * qs[3];
  gqs[1] = (g10 * qs[0] + g11 * qs[1] + g12 * qs[2] + g13 * qs[3]) + g11 * qs[1];
  gqs[2] = (g20 * qs[0] + g22 * qs[2] + g23 * qs[3]) + (g12 * qs[1] + g22 * qs[2]);
  gqs[3] = (g30 * qs[0] + g33 * qs[3]) + (g13 * qs[1] + g23 * qs[2] + g33 * qs[3]);
  float gs = gqs[0] * q[0] + gqs[1] * q[1] + gqs[2] * q[2] + gqs[3] * q[3];
  float gn = gs * (-s / (2.f * n));
#pragma unroll
  for (int k = 0; k < 4; ++k) gq[k] = gqs[k] * s + gn * 2.f * q[k];
}

__global__ void k_quat_fwd(const float* __restrict__ q, long long N, float* __restrict__ R) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float qq[4] = {q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]};
  float r[9];
  quat_to_rot(qq, r);
  float* o = R + 16 * i;
  o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = 0.f;
  o[4] = r[3]; o[5] = r[4]; o[6] = r[5]; o[7] = 0.f;
  o[8] = r[6]; o[9] = r[7]; o[10] = r[8]; o[11] = 0.f;
  o[12] = 0.f; o[13] = 0.f; o[14] = 0.f; o[15] = 1.f;
}

__global__ void k_quat_bwd(const float* __restrict__ gR, const float* __restrict__ q, long long N,
                           float* __restrict__ gq) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float qq[4] = {q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]};
  const float* g = gR + 16 * i;
  float g9[9] = {g[0], g[1], g[2], g[4], g[5], g[6], g[8], g[9], g[10]};
  float out[4];
  quat_bwd(qq, g9, out);
#pragma unroll
  for (int k = 0; k < 4; ++k) gq[4 * i + k] = out[k];
}

__global__ void k_compose(const float* __restrict__ R, const float* __restrict__ t, long long N,
                          float* __restrict__ T) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float* o = T + 16 * i;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[4 * r + c] = R ? R[9 * i + 3 * r + c] : (r == c ? 1.f : 0.f);
    o[4 * r + 3] = t ? t[3 * i + r] : 0.f;
  }
  o[12] = 0.f; o[13] = 0.f; o[14] = 0.f; o[15] = 1.f;
}

// out[m,p,:] = (T[m] @ [points[p],1])[:3]
__global__ void k_tp_fwd(const float* __restrict__ points, long long P, const float* __restrict__ T,
                         long long M, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * P) return;
  long long m = i / P, p = i - m * P;
  const float* t = T + 16 * m;
  float x = points[3 * p], y = points[3 * p + 1], z = points[3 * p + 2];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    out[3 * i + r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[4 * r], x), __fmul_rn(t[4 * r + 1], y)),
                                         __fmul_rn(t[4 * r + 2], z)), t[4 * r + 3]);
}

// gpoints[p] = sum_m R_m^T gout[m,p];  gT[m][:3,:] = sum_p gout[m,p] (x) [points[p],1]
__global__ void k_tp_bwd_points(const float* __restrict__ gout, long long P,
                                const float* __restrict__ T, long long M,
                                float* __restrict__ gpoints) {
  long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float ax = 0.f, ay = 0.f, az = 0.f;
  for (long long m = 0; m < M; ++m) {
    const float* t = T + 16 * m;
    const float* g = gout + 3 * (m * P + p);
    ax += t[0] * g[0] + t[4] * g[1] + t[8] * g[2];
    ay += t[1] * g[0] + t[5] * g[1] + t[9] * g[2];
    az += t[2] * g[0] + t[6] * g[1] + t[10] * g[2];
  }
  gpoints[3 * p] = ax; gpoints[3 * p + 1] = ay; gpoints[3 * p + 2] = az;
}

// one CTA per transform m: deterministic tree reduction of 12 sums over P
__global__ void __launch_bounds__(256)
k_tp_bwd_T(const float* __restrict__ gout, const float* __restrict__ points, long long P,
           float* __restrict__ gT) {
  long long m = blockIdx.x;
  float acc[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) acc[k] = 0.f;
  for (long long p = threadIdx.x; p < P; p += blockDim.x) {
    const float* g = gout + 3 * (m * P + p);
    float x = points[3 * p], y = points[3 * p + 1], z = points[3 * p + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      acc[4 * r + 0] += g[r] * x;
      acc[4 * r + 1] += g[r] * y;
      acc[4 * r + 2] += g[r] * z;
      acc[4 * r + 3] += g[r];
    }
  }
  __shared__ float s[8][12];
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    float v = warp_sum(acc[k]);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    int k = threadIdx.x;
    float v = 0.f;
    if (k < 12)
      for (int w = 0; w < 8; ++w) v += s[w][k];
    gT[16 * m + k] = (k < 12) ? v : 0.f;
  }
}

}  // namespace mf

using namespace mf;

extern "C" int mf_quaternion_matrix_fwd(const float* q, int64_t n, float* R, void* stream_) {
  if (n < 0) return MF_E_BADARG;
  if (n == 0) return MF_OK;
  if (!q || !R) return MF_E_BADARG;
  k_quat_fwd<<<div_up(n, 128), 128, 0, (cudaStream_t)stream_>>>(q, n, R);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
extern "C" int mf_quaternion_matrix_bwd(const float* gR, const float* q, int64_t n, float* gq,
                                        void* stream_) {
  if (n < 0) return MF_E_BADARG;
  if (n == 0) return MF_OK;
  if (!gR || !q || !gq) return MF_E_BADARG;
  k_quat_bwd<<<div_up(n, 128), 128, 0, (cudaStream_t)stream_>>>(gR, q, n, gq);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
extern "C" int mf_compose_transform_fwd(const float* R, const float* t, int64_t n, float* T,
                                        void* stream_) {
  if (n < 0) return MF_E_BADARG;
  if (n == 0) return MF_OK;
  if (!T) return MF_E_BADARG;
  k_compose<<<div_up(n, 128), 128, 0, (cudaStream_t)stream_>>>(R, t, n, T);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
extern "C" int mf_transform_points_fwd(const float* points, int64_t P, const float* T, int64_t M,
                                       float* out, void* stream_) {
  if (P < 0 || M < 0) return MF_E_BADARG;
  if (P == 0 || M == 0) return MF_OK;
  if (!points || !T || !out) return MF_E_BADARG;
  k_tp_fwd<<<div_up(P * M, 256), 256, 0, (cudaStream_t)stream_>>>(points, P, T, M, out);
  MF_LAUNCH_CHECK();
  return MF_OK;
}
extern "C" int mf_transform_points_bwd(const float* gout, const float* points, int64_t P,
                                       const float* T, int64_t M, float* gpoints, float* gT,
                                       void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (P < 0 || M < 0) return MF_E_BADARG;
  if (P == 0 || M == 0) {
    // empty sums: both gradients are zero, not whatever the caller's buffers held
    if (gT && M > 0) MF_CUDA_TRY(cudaMemsetAsync(gT, 0, (size_t)M * 64, stream));
    if (gpoints && P > 0) MF_CUDA_TRY(cudaMemsetAsync(gpoints, 0, (size_t)P * 12, stream));
    return MF_OK;
  }
  if (!gout || !points || !T) return MF_E_BADARG;
  if (gpoints) {
    k_tp_bwd_points<<<div_up(P, 256), 256, 0, stream>>>(gout, P, T, M, gpoints);
    MF_LAUNCH_CHECK();
  }
  if (gT) {
    k_tp_bwd_T<<<(unsigned)M, 256, 0, stream>>>(gout, points, P, gT);
    MF_LAUNCH_CHECK();
  }
  return MF_OK;
}

extern "C" int mf_abi_version(void) { return 1; }
extern "C" int mf_device_sm_count(int device) {
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return -1;
  return n;
}
