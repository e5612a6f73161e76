// Imitation evaluation metrics of IMAmpAgent's sweep (phc/learning/im_amp.py:244-363 + smpl_sim's compute_metrics_lite) accumulated on the
// device, one launch per eval step and one warp per env.  The reference copies body_pos / body_pos_gt of every step to the host, slices
// them per clip ([:num_steps - 1]) and runs numpy over the concatenation; here each env keeps fp64 running sums of the per-frame
// joint means of the five errors and their frame counts, so a clip's contribution is ready when its batch ends:
//   mpjpe_g    |d_t[j]|                                   d_t = pred_t - gt_t (global positions)
//   mpjpe_l    |d_t[j] - d_t[0]|                          root-relative
//   mpjpe_pa   |a R^T y0_j + mu_gt - gt_t[j]|             per-frame similarity alignment of pred onto gt (VideoPose3D's p_mpjpe)
//   vel_dist   |d_t[j] - d_{t-1}[j]|                      = (p_t - p_{t-1}) - (g_t - g_{t-1}); frames t >= 1
//   accel_dist |d_t[j] - 2 d_{t-1}[j] + d_{t-2}[j]|       frames t >= 2
// A frame counts while t < num_steps - 1 (the reference's slice).  d_t goes to a two-slot ring on every step, counted or not; the
// t >= 1 / t >= 2 conditions make a reset of the ring at a batch boundary unnecessary.
//
// The alignment: the rotation that best maps the centred pred onto the centred gt is found with Horn's quaternion method -- the top
// eigenvector of the symmetric 4x4 matrix built from the cross-covariance S = sum_j y0_j x0_j^T, by cyclic Jacobi in fp64.  Its
// eigenvalue is the sign-fixed sum of singular values of the SVD form (so the reflection case needs no special handling) and the
// scale is a = lambda / |y0|^2.  Every lane runs the (warp-uniform) solve on the same butterfly-reduced sums, so no broadcast is
// needed and the result does not depend on the lane.  All reductions are fixed-order shuffles: results are bit-identical run to run.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/phc_b200.h"

namespace phc {
namespace evalm {

constexpr int kWarps = 4;                  // envs per CTA
constexpr int kSlots = 2;                  // bodies per lane: J <= 64
constexpr int kSweeps = 6;                 // Jacobi sweeps of the 4x4 solve (a fixed count: the same work for every env)
constexpr int kFields = PHC_EVAL_ACC_FIELDS;

__device__ __forceinline__ double wsum(double v) {       // every lane ends with the same bits (fp addition commutes)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }

// one Jacobi rotation zeroing A[p][q] (A symmetric 4x4, V accumulates the eigenvectors as columns)
template <int p, int q>
__device__ __forceinline__ void jacobi_rot(double (&A)[4][4], double (&V)[4][4]) {
  const double apq = A[p][q];
  if (apq == 0.0) return;
  const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
  const double at = fabs(theta);
  const double t = at > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (at + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
  for (int k = 0; k < 4; ++k) {            // A P
    const double akp = A[k][p], akq = A[k][q];
    A[k][p] = c * akp - s * akq;
    A[k][q] = s * akp + c * akq;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {            // P^T (A P)
    const double apk = A[p][k], aqk = A[q][k];
    A[p][k] = c * apk - s * aqk;
    A[q][k] = s * apk + c * aqk;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {            // V P
    const double vkp = V[k][p], vkq = V[k][q];
    V[k][p] = c * vkp - s * vkq;
    V[k][q] = s * vkp + c * vkq;
  }
}

// largest eigenvalue of the symmetric A and its eigenvector q (first index on ties)
__device__ __forceinline__ double top_eig4(double (&A)[4][4], double (&q)[4]) {
  double V[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) V[i][k] = i == k ? 1.0 : 0.0;
#pragma unroll 1
  for (int sweep = 0; sweep < kSweeps; ++sweep) {
    jacobi_rot<0, 1>(A, V); jacobi_rot<0, 2>(A, V); jacobi_rot<0, 3>(A, V);
    jacobi_rot<1, 2>(A, V); jacobi_rot<1, 3>(A, V); jacobi_rot<2, 3>(A, V);
  }
  double lam = A[0][0];
#pragma unroll
  for (int k = 0; k < 4; ++k) q[k] = V[k][0];
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (A[i][i] > lam) {
      lam = A[i][i];
#pragma unroll
      for (int k = 0; k < 4; ++k) q[k] = V[k][i];
    }
  return lam;
}

// ring: [2, n, J, 3] (slot t & 1 receives d_t and holds d_{t-2} before that); acc: [n, kFields] fp64, see PHC_EVAL_ACC_FIELDS
__global__ void __launch_bounds__(kWarps * 32)
eval_metrics_kernel(const float* __restrict__ pos, int64_t env_stride, int64_t body_stride, const float* __restrict__ gt,
                    const int32_t* __restrict__ num_steps, int32_t t, int64_t n, int32_t J, float* ring, double* acc) {
  const int lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (e >= n) return;
  const size_t slot = (size_t)n * J * 3;
  float* ring_t = ring + (size_t)(t & 1) * slot + (size_t)e * J * 3;         // d_t goes here; d_{t-2} was here
  const float* ring_1 = ring + (size_t)((t + 1) & 1) * slot + (size_t)e * J * 3;   // d_{t-1}
  float p[kSlots][3], g[kSlots][3], d[kSlots][3], d1[kSlots][3], d2[kSlots][3];
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const int j = lane + 32 * s;
    const bool ok = j < J;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      p[s][c] = ok ? pos[e * env_stride + (int64_t)j * body_stride + c] : 0.0f;
      g[s][c] = ok ? gt[((size_t)e * J + j) * 3 + c] : 0.0f;
      d[s][c] = p[s][c] - g[s][c];
      d1[s][c] = (ok && t >= 1) ? ring_1[j * 3 + c] : 0.0f;
      d2[s][c] = (ok && t >= 2) ? ring_t[j * 3 + c] : 0.0f;
    }
  }
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {       // every lane rewrites only the elements it has just read
    const int j = lane + 32 * s;
    if (j < J)
#pragma unroll
      for (int c = 0; c < 3; ++c) ring_t[j * 3 + c] = d[s][c];
  }
  if (!(t < num_steps[e] - 1)) return;     // outside the clip's counted frames (warp-uniform)

  // root-relative error: d_t[0] lives in lane 0, slot 0
  const float r0x = __shfl_sync(0xffffffffu, d[0][0], 0), r0y = __shfl_sync(0xffffffffu, d[0][1], 0), r0z = __shfl_sync(0xffffffffu, d[0][2], 0);
  double eg = 0.0, el = 0.0, ev = 0.0, ea = 0.0;
  double sp[3] = {0.0, 0.0, 0.0}, sg[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    if (lane + 32 * s >= J) continue;
    const double dx = d[s][0], dy = d[s][1], dz = d[s][2];
    eg += norm3(dx, dy, dz);
    el += norm3(dx - (double)r0x, dy - (double)r0y, dz - (double)r0z);
    ev += norm3(dx - (double)d1[s][0], dy - (double)d1[s][1], dz - (double)d1[s][2]);
    ea += norm3(dx - 2.0 * (double)d1[s][0] + (double)d2[s][0], dy - 2.0 * (double)d1[s][1] + (double)d2[s][1],
                dz - 2.0 * (double)d1[s][2] + (double)d2[s][2]);
#pragma unroll
    for (int c = 0; c < 3; ++c) { sp[c] += (double)p[s][c]; sg[c] += (double)g[s][c]; }
  }
  eg = wsum(eg); el = wsum(el); ev = wsum(ev); ea = wsum(ea);
  const double inv_j = 1.0 / (double)J;
  double mp[3], mg[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { mp[c] = wsum(sp[c]) * inv_j; mg[c] = wsum(sg[c]) * inv_j; }

  // Procrustes: y0 = centred pred, x0 = centred gt; S[a][b] = sum_j y0_a x0_b, yy = sum_j |y0|^2
  double y0[kSlots][3], x0[kSlots][3], S[3][3], yy = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) S[a][b] = 0.0;
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const bool ok = lane + 32 * s < J;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      y0[s][c] = ok ? (double)p[s][c] - mp[c] : 0.0;
      x0[s][c] = ok ? (double)g[s][c] - mg[c] : 0.0;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) S[a][b] += y0[s][a] * x0[s][b];
    yy += y0[s][0] * y0[s][0] + y0[s][1] * y0[s][1] + y0[s][2] * y0[s][2];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) S[a][b] = wsum(S[a][b]);
  yy = wsum(yy);
  // Horn's matrix: its top eigenvector (w, x, y, z) is the unit quaternion of the rotation Q with Q y0_j ~ x0_j
  double N[4][4] = {
      {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0]},
      {S[1][2] - S[2][1], S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2]},
      {S[2][0] - S[0][2], S[0][1] + S[1][0], -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1]},
      {S[0][1] - S[1][0], S[2][0] + S[0][2], S[1][2] + S[2][1], -S[0][0] - S[1][1] + S[2][2]}};
  double qv[4];
  const double lam = top_eig4(N, qv);
  const double qn = 1.0 / (qv[0] * qv[0] + qv[1] * qv[1] + qv[2] * qv[2] + qv[3] * qv[3]);
  const double w = qv[0], x = qv[1], y = qv[2], z = qv[3];
  const double Q[3][3] = {{1.0 - 2.0 * (y * y + z * z) * qn, 2.0 * (x * y - w * z) * qn, 2.0 * (x * z + w * y) * qn},
                          {2.0 * (x * y + w * z) * qn, 1.0 - 2.0 * (x * x + z * z) * qn, 2.0 * (y * z - w * x) * qn},
                          {2.0 * (x * z - w * y) * qn, 2.0 * (y * z + w * x) * qn, 1.0 - 2.0 * (x * x + y * y) * qn}};
  const double scale = lam / yy;
  double epa = 0.0;
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    if (lane + 32 * s >= J) continue;
    double r[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) r[a] = scale * (Q[a][0] * y0[s][0] + Q[a][1] * y0[s][1] + Q[a][2] * y0[s][2]) - x0[s][a];
    epa += norm3(r[0], r[1], r[2]);
  }
  epa = wsum(epa);

  if (lane == 0) {
    double* row = acc + (size_t)e * kFields;
    row[0] += eg * inv_j;
    row[1] += el * inv_j;
    row[2] += epa * inv_j;
    row[5] += 1.0;
    if (t >= 1) { row[3] += ev * inv_j; row[6] += 1.0; }
    if (t >= 2) { row[4] += ea * inv_j; row[7] += 1.0; }
  }
}

}  // namespace evalm
}  // namespace phc

extern "C" void phc_set_error(const char* msg);
extern "C" int phc_check_cuda(cudaError_t e, const char* what);
extern "C" void phc_count_launches(int n);

extern "C" int phc_eval_metrics_step(const float* body_pos, int64_t env_stride, int64_t body_stride, int64_t coord_stride,
                                     const float* body_pos_gt, const int32_t* num_steps, int32_t t, int64_t n, int32_t num_bodies,
                                     float* ring, double* acc, void* stream) {
  using namespace phc::evalm;
  if (n <= 0) { phc_set_error("phc_eval_metrics_step: n <= 0"); return PHC_ERR_INVALID_ARG; }
  if (num_bodies < 1 || num_bodies > 32 * kSlots) {
    phc_set_error("phc_eval_metrics_step: num_bodies must be in [1, 64]"); return PHC_ERR_INVALID_ARG;
  }
  if (coord_stride != 1) { phc_set_error("phc_eval_metrics_step: the x, y, z of a body must be contiguous (coord_stride == 1)"); return PHC_ERR_INVALID_ARG; }
  if (body_stride < 3 || env_stride < (int64_t)num_bodies * body_stride) {
    phc_set_error("phc_eval_metrics_step: bad strides (body_stride >= 3, env_stride >= num_bodies * body_stride)"); return PHC_ERR_INVALID_ARG;
  }
  if (t < 0) { phc_set_error("phc_eval_metrics_step: t < 0"); return PHC_ERR_INVALID_ARG; }
  if (!body_pos || !body_pos_gt || !num_steps || !ring || !acc) {
    phc_set_error("phc_eval_metrics_step: a required pointer is NULL"); return PHC_ERR_INVALID_ARG;
  }
  eval_metrics_kernel<<<(unsigned)((n + kWarps - 1) / kWarps), kWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      body_pos, env_stride, body_stride, body_pos_gt, num_steps, t, n, num_bodies, ring, acc);
  phc_count_launches(1);
  return phc_check_cuda(cudaGetLastError(), "eval_metrics_kernel launch");
}
