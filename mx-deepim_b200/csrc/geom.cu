// geom.cu -- small geometry kernels (compiled with -fmad=false):
//   reprojection-flow labels   lib/flow_c/gpu_flow_kernel.cu:32-69 (flow_kernel) -- the reference's
//                              only native kernel; its host wrapper (l.87-147) does 6 cudaMalloc +
//                              4 H2D + 2 D2H + 6 cudaFree per call, here inputs/outputs stay resident
//   SE(3) compose (float64)    lib/pair_matching/RT_transform.py:127-151 (+ quat2mat l.383-429)
//   ZoomTrans fwd/bwd          deepim/operator_py/zoom_trans.py:22-74
//   Transform3D fwd/bwd        deepim/operator_py/transform3d.py:34-281
//   image transform            lib/utils/image.py:583-594
#include "launch.cuh"

namespace dim {

// ------------------------------------------------------------------------------------------ flow
// HBM-bound: reads depth_src (4 B/px) + a gathered depth_tgt (4 B/px), writes flow (8 B/px) +
// valid (4 B/px) = 20 B/px algorithmic (SURVEY 8(d): 6 144 000 B per 480x640 instance).
__global__ void __launch_bounds__(256) flow_kernel(const float *__restrict__ depth_src,
                                                   const float *__restrict__ depth_tgt,
                                                   const float *__restrict__ KT, float i0, float i1, float i2,
                                                   float i3, float i4, float i5, int H, int W,
                                                   float *__restrict__ flow, float *__restrict__ valid,
                                                   float *__restrict__ valid2 /*nullable: second copy*/) {
  const int b = blockIdx.y;
  const int q4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (q4 >= H * W) return;
  const int h = q4 / W, w0 = q4 % W;
  const size_t P = (size_t)H * W;
  const float *kt = KT + 12 * b;
  const float k0 = kt[0], k1 = kt[1], k2 = kt[2], k3 = kt[3], k4 = kt[4], k5 = kt[5], k6 = kt[6], k7 = kt[7],
              k8 = kt[8], k9 = kt[9], k10 = kt[10], k11 = kt[11];
  const float4 d4 = *reinterpret_cast<const float4 *>(depth_src + (size_t)b * P + q4);
  const float dd[4] = {d4.x, d4.y, d4.z, d4.w};
  float fh[4], fw[4], ok[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int w = w0 + k;
    const float d = dd[k];
    const float x = (((float)w * i0 + (float)h * i1) + i2) * d;
    const float y = (((float)w * i3 + (float)h * i4) + i5) * d;
    const float z = d;
    fh[k] = 0.f; fw[k] = 0.f; ok[k] = 0.f;
    // the reference compares / offsets against DOUBLE literals (gpu_flow_kernel.cu:45,49,56): float operands are promoted
    if ((double)d > 1e-3) {
      const float xp = ((x * k0 + y * k1) + z * k2) + k3;
      const float yp = ((x * k4 + y * k5) + z * k6) + k7;
      const float zp = (float)((double)(((x * k8 + y * k9) + z * k10) + k11) + 1e-15);
      const float wp = xp / zp, hp = yp / zp;
      if (wp >= 0.f && wp <= (float)(W - 1) && hp >= 0.f && hp <= (float)(H - 1)) {
        const int wi = (int)roundf(wp), hi = (int)roundf(hp);
        const float dt = __ldg(depth_tgt + (size_t)b * P + (size_t)hi * W + wi);
        if ((double)fabsf(zp - dt) < 3e-3) {
          fh[k] = hp - (float)h;
          fw[k] = wp - (float)w;
          ok[k] = 1.f;
        }
      }
    }
  }
  *reinterpret_cast<float4 *>(flow + ((size_t)b * 2 + 0) * P + q4) = make_float4(fh[0], fh[1], fh[2], fh[3]);
  *reinterpret_cast<float4 *>(flow + ((size_t)b * 2 + 1) * P + q4) = make_float4(fw[0], fw[1], fw[2], fw[3]);
  *reinterpret_cast<float4 *>(valid + (size_t)b * P + q4) = make_float4(ok[0], ok[1], ok[2], ok[3]);
  if (valid2) *reinterpret_cast<float4 *>(valid2 + (size_t)b * P + q4) = make_float4(ok[0], ok[1], ok[2], ok[3]);
}

int flow_launch(dim_ctx *ctx, const float *depth_src, const float *depth_tgt, const float *KT, const float *Kinv,
                int B, float *flow, float *valid, float *valid2, cudaStream_t st) {
  DIM_REQUIRE((ctx->W & 3) == 0, "width must be a multiple of 4");
  flow_kernel<<<dim3(cdiv(ctx->H * ctx->W / 4, 256), B), 256, 0, st>>>(depth_src, depth_tgt, KT, Kinv[0], Kinv[1],
                                                                        Kinv[2], Kinv[3], Kinv[4], Kinv[5], ctx->H,
                                                                        ctx->W, flow, valid, valid2);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------- se3
__device__ __forceinline__ void quat2mat_f64(const double *q, double *M) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double Nq = w * w + x * x + y * y + z * z;
  if (Nq < 2.220446049250313e-16 * 4.0) {  // _FLOAT_EPS (RT_transform.py:236-238)
    M[0] = M[4] = M[8] = 1.0;
    M[1] = M[2] = M[3] = M[5] = M[6] = M[7] = 0.0;
    return;
  }
  const double s = 2.0 / Nq;
  const double X = x * s, Y = y * s, Z = z * s;
  const double wX = w * X, wY = w * Y, wZ = w * Z, xX = x * X, xY = x * Y, xZ = x * Z, yY = y * Y, yZ = y * Z,
               zZ = z * Z;
  M[0] = 1.0 - (yY + zZ); M[1] = xY - wZ;         M[2] = xZ + wY;
  M[3] = xY + wZ;         M[4] = 1.0 - (xX + zZ); M[5] = yZ - wX;
  M[6] = xZ - wY;         M[7] = yZ + wX;         M[8] = 1.0 - (xX + yY);
}

__device__ void rt_transform_f64(const double *ps, const double *quat, const double *td, const double *Tm,
                                 const double *Ts, int rot_coord, double *po) {
  const double n = sqrt(quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2] + quat[3] * quat[3]);
  const double q[4] = {quat[0] / n, quat[1] / n, quat[2] / n, quat[3] / n};
  double Rd[9];
  quat2mat_f64(q, Rd);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 3; ++k)
        acc += (rot_coord == 0) ? ps[i * 4 + k] * Rd[k * 3 + j] : Rd[i * 3 + k] * ps[k * 4 + j];
      po[i * 4 + j] = acc;
    }
  const double d0 = td[0] * Ts[0] + Tm[0], d1 = td[1] * Ts[1] + Tm[1], d2 = td[2] * Ts[2] + Tm[2];
  const double sx = ps[3], sy = ps[7], sz = ps[11];
  const double z2 = sz / exp(d2);
  po[11] = z2;
  if (rot_coord == 2) {
    po[3] = sz * d0 + sx;
    po[7] = sz * d1 + sy;
  } else {
    po[3] = z2 * (d0 + sx / sz);
    po[7] = z2 * (d1 + sy / sz);
  }
}

__global__ void se3_compose_kernel(const double *pose_src, const float *se3, int B, double m0, double m1, double m2,
                                   double s0, double s1, double s2, int rot_coord, double *pose_out,
                                   float *pose_out_f32) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double ps[12], po[12];
  for (int k = 0; k < 12; ++k) ps[k] = pose_src[12 * b + k];
  const double quat[4] = {(double)se3[7 * b], (double)se3[7 * b + 1], (double)se3[7 * b + 2], (double)se3[7 * b + 3]};
  const double td[3] = {(double)se3[7 * b + 4], (double)se3[7 * b + 5], (double)se3[7 * b + 6]};
  const double Tm[3] = {m0, m1, m2}, Ts[3] = {s0, s1, s2};
  rt_transform_f64(ps, quat, td, Tm, Ts, rot_coord, po);
  for (int k = 0; k < 12; ++k) {
    pose_out[12 * b + k] = po[k];
    if (pose_out_f32) pose_out_f32[12 * b + k] = (float)po[k];
  }
}

int se3_compose_launch(const double *pose_src, const float *se3, int B, const double *Tm, const double *Ts,
                       int rot_coord, double *pose_out, float *pose_out_f32, cudaStream_t st) {
  se3_compose_kernel<<<cdiv(B, 64), 64, 0, st>>>(pose_src, se3, B, Tm[0], Tm[1], Tm[2], Ts[0], Ts[1], Ts[2],
                                                  rot_coord, pose_out, pose_out_f32);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------- train-time pose / label update
// lib/pair_matching/batch_updater_py_multi.py:174-259 per instance: refined pose = RT_transform(src,
// rot_est, trans_est); new labels (rot as quaternion via mat2quat, trans) = calc_RT_delta(refined, tgt,
// "QUAT"); KT = K . calc_se3(refined, tgt) for the reprojection-flow kernel.
// mat2quat (RT_transform.py:432-509) takes the eigenvector of the largest eigenvalue of a symmetric 4x4
// matrix (numpy eigh); here a cyclic Jacobi iteration in float64.
__device__ void jacobi_eig4(double A[4][4], double V[4][4]) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 24; ++sweep) {
    double off = 0.0;
    for (int p_ = 0; p_ < 3; ++p_)
      for (int q = p_ + 1; q < 4; ++q) off += A[p_][q] * A[p_][q];
    if (off < 1e-32) break;
    for (int p_ = 0; p_ < 3; ++p_)
      for (int q = p_ + 1; q < 4; ++q) {
        if (fabs(A[p_][q]) < 1e-300) continue;
        const double theta = (A[q][q] - A[p_][p_]) / (2.0 * A[p_][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
        for (int k = 0; k < 4; ++k) {
          const double akp = A[k][p_], akq = A[k][q];
          A[k][p_] = c * akp - sn * akq;
          A[k][q] = sn * akp + c * akq;
        }
        for (int k = 0; k < 4; ++k) {
          const double apk = A[p_][k], aqk = A[q][k];
          A[p_][k] = c * apk - sn * aqk;
          A[q][k] = sn * apk + c * aqk;
        }
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p_], vkq = V[k][q];
          V[k][p_] = c * vkp - sn * vkq;
          V[k][q] = sn * vkp + c * vkq;
        }
      }
  }
}

__device__ void mat2quat_f64(const double *M, double *q) {
  const double Qxx = M[0], Qyx = M[1], Qzx = M[2], Qxy = M[3], Qyy = M[4], Qzy = M[5], Qxz = M[6], Qyz = M[7],
               Qzz = M[8];
  double A[4][4] = {{Qxx - Qyy - Qzz, Qyx + Qxy, Qzx + Qxz, Qyz - Qzy},
                    {Qyx + Qxy, Qyy - Qxx - Qzz, Qzy + Qyz, Qzx - Qxz},
                    {Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, Qxy - Qyx},
                    {Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz}};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) A[i][j] /= 3.0;
  double V[4][4];
  jacobi_eig4(A, V);
  int best = 0;
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > A[best][best]) best = k;
  q[0] = V[3][best]; q[1] = V[0][best]; q[2] = V[1][best]; q[3] = V[2][best];
  if (q[0] < 0)
    for (int k = 0; k < 4; ++k) q[k] = -q[k];
}

__global__ void train_pose_kernel(const float *src_pose, const float *rot_est, const float *trans_est,
                                  const float *tgt_pose, int B, double m0, double m1, double m2, double s0, double s1,
                                  double s2, int rot_coord, double k0, double k1, double k2, double k3, double k4,
                                  double k5, double k6, double k7, double k8, float *pose_new_f32, float *rot_label,
                                  float *trans_label, float *KT, float *light_pos, double l0, double l1, double l2) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double ps[12], pt[12], po[12];
  for (int k = 0; k < 12; ++k) { ps[k] = (double)src_pose[12 * b + k]; pt[k] = (double)tgt_pose[12 * b + k]; }
  const double quat[4] = {(double)rot_est[4 * b], (double)rot_est[4 * b + 1], (double)rot_est[4 * b + 2],
                          (double)rot_est[4 * b + 3]};
  const double td[3] = {(double)trans_est[3 * b], (double)trans_est[3 * b + 1], (double)trans_est[3 * b + 2]};
  const double Tm[3] = {m0, m1, m2}, Ts[3] = {s0, s1, s2};
  rt_transform_f64(ps, quat, td, Tm, Ts, rot_coord, po);
  for (int k = 0; k < 12; ++k) pose_new_f32[12 * b + k] = (float)po[k];
  // ModelNet branch (batch_updater_py_multi.py:203-207): the light follows the float64 refined pose
  if (light_pos) {
    light_pos[3 * b + 0] = (float)(l0 + po[3]);
    light_pos[3 * b + 1] = (float)(l1 - po[7]);
    light_pos[3 * b + 2] = (float)(l2 - po[11]);
  }
  // calc_RT_delta(refined, tgt, QUAT)  (RT_transform.py:16-44)
  double Rd[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
      for (int k = 0; k < 3; ++k) acc += (rot_coord == 0) ? po[k * 4 + i] * pt[k * 4 + j] : pt[i * 4 + k] * po[j * 4 + k];
      Rd[i * 3 + j] = acc;
    }
  double q[4];
  mat2quat_f64(Rd, q);
  for (int k = 0; k < 4; ++k) rot_label[4 * b + k] = (float)q[k];
  double d[3];
  if (rot_coord == 2) {
    d[0] = (pt[3] - po[3]) / po[11];
    d[1] = (pt[7] - po[7]) / po[11];
  } else {
    // tgt_pose is a float32 array in the train loop: T_tgt[0]/T_tgt[2] is a float32 division
    const float *tg32 = tgt_pose + 12 * b;
    d[0] = (double)(tg32[3] / tg32[11]) - po[3] / po[11];
    d[1] = (double)(tg32[7] / tg32[11]) - po[7] / po[11];
  }
  d[2] = log(po[11] / pt[11]);
  for (int k = 0; k < 3; ++k) trans_label[3 * b + k] = (float)((d[k] - Tm[k]) / Ts[k]);
  // calc_se3 (RT_transform.py:176-187 over lib/utils/projection.py: float32 storage) then K . se3
  float Ri[9], Ti[3];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Ri[i * 3 + j] = (float)po[j * 4 + i];
    Ti[i] = (float)(-1.0 * ((po[0 * 4 + i] * po[3] + po[1 * 4 + i] * po[7]) + po[2 * 4 + i] * po[11]));
  }
  const float *tg = tgt_pose + 12 * b;
  float se3[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      se3[i * 4 + j] = (tg[i * 4 + 0] * Ri[0 * 3 + j] + tg[i * 4 + 1] * Ri[1 * 3 + j]) + tg[i * 4 + 2] * Ri[2 * 3 + j];
    se3[i * 4 + 3] = ((tg[i * 4 + 0] * Ti[0] + tg[i * 4 + 1] * Ti[1]) + tg[i * 4 + 2] * Ti[2]) + tg[i * 4 + 3];
  }
  const double Kd[9] = {k0, k1, k2, k3, k4, k5, k6, k7, k8};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j)
      KT[12 * b + i * 4 + j] = (float)((Kd[i * 3 + 0] * (double)se3[0 * 4 + j] + Kd[i * 3 + 1] * (double)se3[1 * 4 + j]) +
                                        Kd[i * 3 + 2] * (double)se3[2 * 4 + j]);
}

// light_pos (nullable) [B,3]: also write the light of the ModelNet branch, light_offset + (t_x, -t_y, -t_z) of the refined pose
int train_pose_launch(const float *src_pose, const float *rot_est, const float *trans_est, const float *tgt_pose, int B,
                      const double *Tm, const double *Ts, int rot_coord, const double *K9, float *pose_new_f32,
                      float *rot_label, float *trans_label, float *KT, cudaStream_t st, float *light_pos,
                      const double *light_offset) {
  const double l0 = light_pos ? light_offset[0] : 0.0, l1 = light_pos ? light_offset[1] : 0.0,
               l2 = light_pos ? light_offset[2] : 0.0;
  train_pose_kernel<<<cdiv(B, 32), 32, 0, st>>>(src_pose, rot_est, trans_est, tgt_pose, B, Tm[0], Tm[1], Tm[2], Ts[0],
                                                 Ts[1], Ts[2], rot_coord, K9[0], K9[1], K9[2], K9[3], K9[4], K9[5], K9[6],
                                                 K9[7], K9[8], pose_new_f32, rot_label, trans_label, KT, light_pos, l0, l1,
                                                 l2);
  DIM_LAUNCH_CHECK();
  return 0;
}

__global__ void f64_to_f32_kernel(const double *a, float *b, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = (float)a[i];
}
int f64_to_f32_launch(const double *a, float *b, int n, cudaStream_t st) {
  f64_to_f32_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, b, n);
  DIM_LAUNCH_CHECK();
  return 0;
}

// Per-iteration head of the lit refinement chain (ModelNet branch, deepim/core/tester.py:146-160): the float32 src_pose blob
// (as f64_to_f32) and the light that follows the pose, light = float32(offset[0] + t_x, offset[1] - t_y, offset[2] - t_z)
// evaluated on the FLOAT64 pose before the cast (numpy float64 arithmetic; glumpy casts the uniform to float32).
__global__ void pose_light_kernel(const double *pose, float *pose_f32, float *light_pos, int B, double o0, double o1,
                                  double o2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 12 * B) pose_f32[i] = (float)pose[i];
  if (i < B) {
    const double *p = pose + 12 * i;
    light_pos[3 * i + 0] = (float)(o0 + p[3]);
    light_pos[3 * i + 1] = (float)(o1 - p[7]);
    light_pos[3 * i + 2] = (float)(o2 - p[11]);
  }
}
int pose_light_launch(const double *pose, float *pose_f32, float *light_pos, int B, const double *offset, cudaStream_t st) {
  pose_light_kernel<<<cdiv(12 * B, 256), 256, 0, st>>>(pose, pose_f32, light_pos, B, offset[0], offset[1], offset[2]);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------ ZoomTrans
__global__ void zoom_trans_kernel(const float *zoom_factor, const float *in, int B, int mul, int scale_xy,
                                  float *out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float w = zoom_factor[4 * b];
  const float x = in[3 * b], y = in[3 * b + 1], z = in[3 * b + 2];
  out[3 * b + 0] = scale_xy ? (mul ? x * w : x / w) : x;
  out[3 * b + 1] = scale_xy ? (mul ? y * w : y / w) : y;
  out[3 * b + 2] = z;
}
int zoom_trans_launch(const float *zoom_factor, const float *in, int B, int mul, int scale_xy, float *out,
                      cudaStream_t st) {
  zoom_trans_kernel<<<cdiv(B, 64), 64, 0, st>>>(zoom_factor, in, B, mul, scale_xy, out);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------- Transform3D
// quat2mat_forward (transform3d.py:185-212): identity unless |Nq-1| < 1e-2; float32 inputs, the
// python arithmetic promotes to float64, result stored float32.
__device__ __forceinline__ void quat2mat_fwd_t3d(const float *q, float *M) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  const float Nq = w * w + x * x + y * y + z * z;
  const double dn = (double)Nq - 1.0;
  if (!(-1e-2 < dn && dn < 1e-2)) {
    M[0] = M[4] = M[8] = 1.f;
    M[1] = M[2] = M[3] = M[5] = M[6] = M[7] = 0.f;
    return;
  }
  const double s = 2.0 / (double)Nq;
  const double X = x * s, Y = y * s, Z = z * s;
  const double wX = w * X, wY = w * Y, wZ = w * Z, xX = x * X, xY = x * Y, xZ = x * Z, yY = y * Y, yZ = y * Z,
               zZ = z * Z;
  M[0] = (float)(1.0 - (yY + zZ)); M[1] = (float)(xY - wZ);         M[2] = (float)(xZ + wY);
  M[3] = (float)(xY + wZ);         M[4] = (float)(1.0 - (xX + zZ)); M[5] = (float)(yZ - wX);
  M[6] = (float)(xZ - wY);         M[7] = (float)(yZ + wX);         M[8] = (float)(1.0 - (xX + yY));
}

struct T3DParams {
  const float *points, *rotation, *translation, *pose_src;
  int B, N, rot_coord;
  float Tm[3], Ts[3];
};

__device__ __forceinline__ void t3d_pose(const T3DParams &p, int b, float *Rt, float *Tt, float *Rd_out) {
  float Rd[9];
  quat2mat_fwd_t3d(p.rotation + 4 * b, Rd);
  const float *ps = p.pose_src + 12 * b;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      float acc = 0.f;
      for (int k = 0; k < 3; ++k)
        acc += (p.rot_coord == 0) ? ps[i * 4 + k] * Rd[k * 3 + j] : Rd[i * 3 + k] * ps[k * 4 + j];
      Rt[i * 3 + j] = acc;
    }
  const float *td = p.translation + 3 * b;
  const float d0 = td[0] * p.Ts[0] + p.Tm[0], d1 = td[1] * p.Ts[1] + p.Tm[1], d2 = td[2] * p.Ts[2] + p.Tm[2];
  const float sx = ps[3], sy = ps[7], sz = ps[11];
  const float z2 = sz / expf(d2);
  Tt[2] = z2;
  if (p.rot_coord == 2) {
    Tt[0] = sz * d0 + sx;
    Tt[1] = sz * d1 + sy;
  } else {
    Tt[0] = z2 * (d0 + sx / sz);
    Tt[1] = z2 * (d1 + sy / sz);
  }
  if (Rd_out)
    for (int k = 0; k < 9; ++k) Rd_out[k] = Rd[k];
}

__global__ void __launch_bounds__(256) transform3d_fwd_kernel(T3DParams p, float *out) {
  const int b = blockIdx.y;
  __shared__ float Rt[9], Tt[3];
  if (threadIdx.x == 0) t3d_pose(p, b, Rt, Tt, nullptr);
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.N) return;
  const float *pc = p.points + (size_t)b * 3 * p.N;
  const float x = pc[n], y = pc[p.N + n], z = pc[2 * p.N + n];
  float *o = out + (size_t)b * 3 * p.N;
  o[n] = ((Rt[0] * x + Rt[1] * y) + Rt[2] * z) + Tt[0];
  o[p.N + n] = ((Rt[3] * x + Rt[4] * y) + Rt[5] * z) + Tt[1];
  o[2 * p.N + n] = ((Rt[6] * x + Rt[7] * y) + Rt[8] * z) + Tt[2];
}

// backward (transform3d.py:99-281): one block per instance reduces sum_n D (3) and D.P^T (3x3)
__global__ void __launch_bounds__(256) transform3d_bwd_kernel(T3DParams p, const float *out_grad, float *rot_grad,
                                                              float *trans_grad) {
  const int b = blockIdx.x;
  const float *D = out_grad + (size_t)b * 3 * p.N;
  const float *pc = p.points + (size_t)b * 3 * p.N;
  float acc[12];
  for (int k = 0; k < 12; ++k) acc[k] = 0.f;
  for (int n = threadIdx.x; n < p.N; n += blockDim.x) {
    const float d[3] = {D[n], D[p.N + n], D[2 * p.N + n]};
    const float q[3] = {pc[n], pc[p.N + n], pc[2 * p.N + n]};
    for (int i = 0; i < 3; ++i) {
      acc[i] += d[i];
      for (int j = 0; j < 3; ++j) acc[3 + i * 3 + j] += d[i] * q[j];
    }
  }
  __shared__ float red[12][8];
  for (int k = 0; k < 12; ++k) {
    float v = acc[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  float s[12];
  for (int k = 0; k < 12; ++k) {
    s[k] = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s[k] += red[k][w];
  }
  const float *Dt = s;       // T_tgt_diff (3)
  const float *RtD = s + 3;  // Rm_tgt_diff (3x3)
  const float *ps = p.pose_src + 12 * b;
  // --- T_transform_backward (transform3d.py:153-183)
  {
    const float *td = p.translation + 3 * b;
    const float d0 = td[0] * p.Ts[0] + p.Tm[0], d1 = td[1] * p.Ts[1] + p.Tm[1], d2 = td[2] * p.Ts[2] + p.Tm[2];
    const float sx = ps[3], sy = ps[7], sz = ps[11];
    const float z2 = sz / expf(d2);
    float g0, g1, g2;
    if (p.rot_coord == 2) {
      g0 = Dt[0] * (p.Ts[0] * sz);
      g1 = Dt[1] * (p.Ts[1] * sz);
      g2 = Dt[2] * (-p.Ts[2] * z2);
    } else {
      g0 = Dt[0] * (p.Ts[0] * z2);
      g1 = Dt[1] * (p.Ts[1] * z2);
      const float share = -p.Ts[2] * z2;
      g2 = Dt[0] * (share * (d0 + sx / sz)) + Dt[1] * (share * (d1 + sy / sz)) + Dt[2] * (-p.Ts[2] * z2);
    }
    trans_grad[3 * b] = g0; trans_grad[3 * b + 1] = g1; trans_grad[3 * b + 2] = g2;
  }
  // --- Rm_delta_diff: model: Rs^T . RtD ; camera: RtD . Rs^T  (l.127-131)
  float Dm[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      float a = 0.f;
      for (int k = 0; k < 3; ++k)
        a += (p.rot_coord == 0) ? ps[k * 4 + i] * RtD[k * 3 + j] : RtD[i * 3 + k] * ps[j * 4 + k];
      Dm[i * 3 + j] = a;
    }
  // --- quat2mat_backward (l.214-281): zero unless |Nq-1| < 1e-4
  const float *q = p.rotation + 4 * b;
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  const float Nq = w * w + x * x + y * y + z * z;
  const double dn = (double)Nq - 1.0;
  float *rg = rot_grad + 4 * b;
  if (!(-1e-4 < dn && dn < 1e-4)) {
    rg[0] = rg[1] = rg[2] = rg[3] = 0.f;
    return;
  }
  const float Ns = sqrtf(Nq);
  const float w_ = w / Ns, x_ = x / Ns, y_ = y / Ns, z_ = z / Ns;
#define DD(i, j) ((double)Dm[(i)*3 + (j)])
  double wd = -z_ * DD(0, 1) + y_ * DD(0, 2) + z_ * DD(1, 0) - x_ * DD(1, 2) - y_ * DD(2, 0) + x_ * DD(2, 1);
  double xd = y_ * DD(0, 1) + z_ * DD(0, 2) + y_ * DD(1, 0) - 2 * x_ * DD(1, 1) - w_ * DD(1, 2) + z_ * DD(2, 0) +
              w_ * DD(2, 1) - 2 * x_ * DD(2, 2);
  double yd = -2 * y_ * DD(0, 0) + x_ * DD(0, 1) + w_ * DD(0, 2) + x_ * DD(1, 0) + z_ * DD(1, 2) - w_ * DD(2, 0) +
              z_ * DD(2, 1) - 2 * y_ * DD(2, 2);
  double zd = -2 * z_ * DD(0, 0) - w_ * DD(0, 1) + x_ * DD(0, 2) + w_ * DD(1, 0) - 2 * z_ * DD(1, 1) +
              y_ * DD(1, 2) + x_ * DD(2, 0) + y_ * DD(2, 1);
#undef DD
  wd *= 2.0; xd *= 2.0; yd *= 2.0; zd *= 2.0;
  const double Nsd = (double)Ns;
  const double share = Nsd * Nsd * Nsd * (w * wd + x * xd + y * yd + z * zd);
  rg[0] = (float)(Nsd * wd - w * share);
  rg[1] = (float)(Nsd * xd - x * share);
  rg[2] = (float)(Nsd * yd - y * share);
  rg[3] = (float)(Nsd * zd - z * share);
}

static T3DParams make_t3d(const float *pc, const float *rot, const float *tr, const float *ps, int B, int N,
                          const float *Tm, const float *Ts, int rot_coord) {
  T3DParams p;
  p.points = pc; p.rotation = rot; p.translation = tr; p.pose_src = ps; p.B = B; p.N = N; p.rot_coord = rot_coord;
  for (int k = 0; k < 3; ++k) { p.Tm[k] = Tm[k]; p.Ts[k] = Ts[k]; }
  return p;
}

int transform3d_fwd_launch(const float *pc, const float *rot, const float *tr, const float *ps, int B, int N,
                           const float *Tm, const float *Ts, int rot_coord, float *out, cudaStream_t st) {
  T3DParams p = make_t3d(pc, rot, tr, ps, B, N, Tm, Ts, rot_coord);
  transform3d_fwd_kernel<<<dim3(cdiv(N, 256), B), 256, 0, st>>>(p, out);
  DIM_LAUNCH_CHECK();
  return 0;
}
int transform3d_bwd_launch(const float *og, const float *pc, const float *rot, const float *tr, const float *ps,
                           int B, int N, const float *Tm, const float *Ts, int rot_coord, float *rot_grad,
                           float *trans_grad, cudaStream_t st) {
  T3DParams p = make_t3d(pc, rot, tr, ps, B, N, Tm, Ts, rot_coord);
  transform3d_bwd_kernel<<<B, 256, 0, st>>>(p, og, rot_grad, trans_grad);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------ image transform
// u8 BGR HWC -> f32 RGB-mean CHW (lib/utils/image.py:583-594; float64 subtract, float32 store)
__global__ void __launch_bounds__(256) transform_u8_kernel(const uint8_t *bgr, int H, int W, double m0, double m1,
                                                           double m2, float *out) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * W) return;
  const size_t P = (size_t)H * W;
  const uint8_t *px = bgr + ((size_t)b * P + q) * 3;
  float *o = out + (size_t)b * 3 * P;
  o[q] = (float)((double)px[2] - m0);
  o[P + q] = (float)((double)px[1] - m1);
  o[2 * P + q] = (float)((double)px[0] - m2);
}
int transform_u8_launch(dim_ctx *ctx, const uint8_t *bgr, int B, const double *means, float *out, cudaStream_t st) {
  transform_u8_kernel<<<dim3(cdiv(ctx->H * ctx->W, 256), B), 256, 0, st>>>(bgr, ctx->H, ctx->W, means[0], means[1],
                                                                            means[2], out);
  DIM_LAUNCH_CHECK();
  return 0;
}

// u8 BGR HWC -> pixel-interleaved float4 (RGB - mean) + mean (w = 0): dim_refine_host_async's input transform (float64 subtraction
// cast to float32, lib/utils/image.py:583-594) followed by the zoom sampler's float32 "+ mean" (zoom_image_with_factor.py:44)
__global__ void __launch_bounds__(256) transform_u8_obs4_kernel(const uint8_t *bgr, int P, double m0, double m1,
                                                                double m2, float4 *out) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= P) return;
  const uint8_t *px = bgr + ((size_t)b * P + q) * 3;
  out[(size_t)b * P + q] = make_float4((float)((double)px[2] - m0) + (float)m0, (float)((double)px[1] - m1) + (float)m1,
                                       (float)((double)px[0] - m2) + (float)m2, 0.f);
}
int transform_u8_obs4_launch(dim_ctx *ctx, const uint8_t *bgr, int B, const double *means, float4 *out, cudaStream_t st) {
  const int P = ctx->H * ctx->W;
  transform_u8_obs4_kernel<<<dim3(cdiv(P, 256), B), 256, 0, st>>>(bgr, P, means[0], means[1], means[2], out);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------- ADD / ADI
// lib/utils/pose_error.py:72-108 in float64: ADD = mean_p |(R^ p + t^) - (R p + t)|, ADI = mean over the GT-transformed
// points of the distance to the nearest ESTIMATE-transformed point (cKDTree(pts_est).query(pts_gt)): brute force, one block
// per pose pair, the estimate cloud staged through shared memory in tiles.  Fixed-order block reduction (deterministic).
__global__ void __launch_bounds__(256) pose_error_kernel(const double *pose_est, const double *pose_gt, const double *pts, int N,
                                                         int symmetric, double *out) {
  __shared__ double Pe[12], Pg[12];
  __shared__ double tile[256 * 3];
  __shared__ double red[256];
  const int m = blockIdx.x;
  if (threadIdx.x < 12) { Pe[threadIdx.x] = pose_est[12 * m + threadIdx.x]; Pg[threadIdx.x] = pose_gt[12 * m + threadIdx.x]; }
  __syncthreads();
  double acc = 0.0;
  if (!symmetric) {
    for (int n = threadIdx.x; n < N; n += 256) {
      const double x = pts[3 * n], y = pts[3 * n + 1], z = pts[3 * n + 2];
      double d2 = 0.0;
      for (int r = 0; r < 3; ++r) {
        const double e = ((Pe[4 * r] * x + Pe[4 * r + 1] * y) + Pe[4 * r + 2] * z) + Pe[4 * r + 3];
        const double g = ((Pg[4 * r] * x + Pg[4 * r + 1] * y) + Pg[4 * r + 2] * z) + Pg[4 * r + 3];
        d2 += (e - g) * (e - g);
      }
      acc += sqrt(d2);
    }
  } else {
    for (int n0 = 0; n0 < N; n0 += 256) {  // every thread owns GT point n0 + tid; loop over all estimate points by tiles
      const int n = n0 + threadIdx.x;
      double gx = 0, gy = 0, gz = 0;
      if (n < N) {
        const double x = pts[3 * n], y = pts[3 * n + 1], z = pts[3 * n + 2];
        gx = ((Pg[0] * x + Pg[1] * y) + Pg[2] * z) + Pg[3];
        gy = ((Pg[4] * x + Pg[5] * y) + Pg[6] * z) + Pg[7];
        gz = ((Pg[8] * x + Pg[9] * y) + Pg[10] * z) + Pg[11];
      }
      double best = 1e300;
      for (int k0 = 0; k0 < N; k0 += 256) {
        __syncthreads();
        const int k = k0 + threadIdx.x;
        if (k < N) {
          const double x = pts[3 * k], y = pts[3 * k + 1], z = pts[3 * k + 2];
          tile[3 * threadIdx.x] = ((Pe[0] * x + Pe[1] * y) + Pe[2] * z) + Pe[3];
          tile[3 * threadIdx.x + 1] = ((Pe[4] * x + Pe[5] * y) + Pe[6] * z) + Pe[7];
          tile[3 * threadIdx.x + 2] = ((Pe[8] * x + Pe[9] * y) + Pe[10] * z) + Pe[11];
        }
        __syncthreads();
        const int cnt = min(256, N - k0);
        for (int j = 0; j < cnt; ++j) {
          const double dx = tile[3 * j] - gx, dy = tile[3 * j + 1] - gy, dz = tile[3 * j + 2] - gz;
          const double d2 = (dx * dx + dy * dy) + dz * dz;
          best = d2 < best ? d2 : best;
        }
      }
      if (n < N) acc += sqrt(best);
    }
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[m] = red[0] / (double)N;
}
// End-point error of a predicted flow field (deepim/core/tester.py:573-589 calc_EPE_one_pair): per instance the sums of
// |flow_gt - flow_pred| over all pixels / the visible ones / visible-or-background, and the three pixel counts.
// flows [B,2,H,W] (plane order as the graph emits them), visible / bg [B,1,H,W].  out [B,6] float64:
// epe_all, num_all, epe_viz, num_viz, epe_vizbg, num_vizbg.  One block per instance, fixed-order reduction.
__global__ void __launch_bounds__(256) epe_kernel(const float *pred, const float *gt, const float *visible, const float *bg, int P,
                                                  double *out) {
  __shared__ double red[5][256];
  const int b = blockIdx.x;
  const float *p0 = pred + (size_t)b * 2 * P, *g0 = gt + (size_t)b * 2 * P, *v = visible + (size_t)b * P, *bgp = bg + (size_t)b * P;
  double s_all = 0, s_viz = 0, n_viz = 0, s_vb = 0, n_vb = 0;
  for (int q = threadIdx.x; q < P; q += 256) {
    const float dx = g0[q] - p0[q], dy = g0[P + q] - p0[P + q];
    const double d = (double)sqrtf(dx * dx + dy * dy);  // np.sqrt(np.square(x) + np.square(y)) on float32 arrays
    const bool vz = v[q] == 1.0f, vb = (v[q] != 0.0f) || (bgp[q] != 0.0f);
    s_all += d;
    if (vz) s_viz += d;
    n_viz += (double)v[q];
    if (vb) { s_vb += d; n_vb += 1.0; }
  }
  red[0][threadIdx.x] = s_all; red[1][threadIdx.x] = s_viz; red[2][threadIdx.x] = n_viz; red[3][threadIdx.x] = s_vb; red[4][threadIdx.x] = n_vb;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s)
      for (int k = 0; k < 5; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[6 * b] = red[0][0]; out[6 * b + 1] = (double)P; out[6 * b + 2] = red[1][0]; out[6 * b + 3] = red[2][0];
    out[6 * b + 4] = red[3][0]; out[6 * b + 5] = red[4][0];
  }
}
int epe_launch(const float *pred, const float *gt, const float *visible, const float *bg, int B, int P, double *out, cudaStream_t st) {
  epe_kernel<<<B, 256, 0, st>>>(pred, gt, visible, bg, P, out);
  DIM_LAUNCH_CHECK();
  return 0;
}

// Average re-projection error in 2D (lib/utils/pose_error.py:27-69 `arp_2d`: mean_p | proj(K (R^ p + t^)) - proj(K (R p + t)) |,
// pixels) and the rotation / translation distance of LM6D_REFINE.evaluate_pose (lib/pair_matching/RT_transform.py:162-173
// `calc_rt_dist_m`: geodesic angle of R_est^T R_gt in degrees -- the reference's |logm(.)|_F / sqrt(2) -- and |t_gt - t_est|).
// One block per pose pair; out2 = [M,3]: arp_2d, rot_deg, trans_m.  float64, fixed-order reduction.
__global__ void __launch_bounds__(256) pose_error2d_kernel(const double *pose_est, const double *pose_gt, const double *pts, int N,
                                                           const double *K9, double *out3) {
  __shared__ double Pe[12], Pg[12], Kk[9];
  __shared__ double red[256];
  const int m = blockIdx.x;
  if (threadIdx.x < 12) { Pe[threadIdx.x] = pose_est[12 * m + threadIdx.x]; Pg[threadIdx.x] = pose_gt[12 * m + threadIdx.x]; }
  if (threadIdx.x < 9) Kk[threadIdx.x] = K9[threadIdx.x];
  __syncthreads();
  double acc = 0.0;
  for (int n = threadIdx.x; n < N; n += 256) {
    const double x = pts[3 * n], y = pts[3 * n + 1], z = pts[3 * n + 2];
    double e[3], g[3], ce[3], cg[3];
    for (int r = 0; r < 3; ++r) {
      e[r] = ((Pe[4 * r] * x + Pe[4 * r + 1] * y) + Pe[4 * r + 2] * z) + Pe[4 * r + 3];
      g[r] = ((Pg[4 * r] * x + Pg[4 * r + 1] * y) + Pg[4 * r + 2] * z) + Pg[4 * r + 3];
    }
    for (int r = 0; r < 3; ++r) {
      ce[r] = (Kk[3 * r] * e[0] + Kk[3 * r + 1] * e[1]) + Kk[3 * r + 2] * e[2];
      cg[r] = (Kk[3 * r] * g[0] + Kk[3 * r + 1] * g[1]) + Kk[3 * r + 2] * g[2];
    }
    const double du = ce[0] / ce[2] - cg[0] / cg[2], dv = ce[1] / ce[2] - cg[1] / cg[2];
    acc += sqrt(du * du + dv * dv);
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out3[3 * m] = N > 0 ? red[0] / (double)N : 0.0;
    // trace(R_est^T R_gt) = sum_ij R_est[i][j] R_gt[i][j]; the off-diagonal antisymmetric part gives sin for small angles
    double tr = 0.0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) tr += Pe[4 * i + j] * Pg[4 * i + j];
    // M = R_est^T R_gt; sin(theta) = |axis part| = 0.5 * |(M32-M23, M13-M31, M21-M12)|: atan2 keeps precision near 0 and 180
    double Mx[3][3];
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) Mx[a][b] = (Pe[a] * Pg[b] + Pe[4 + a] * Pg[4 + b]) + Pe[8 + a] * Pg[8 + b];
    const double sx = Mx[2][1] - Mx[1][2], sy = Mx[0][2] - Mx[2][0], sz = Mx[1][0] - Mx[0][1];
    const double sn = 0.5 * sqrt((sx * sx + sy * sy) + sz * sz), cs = 0.5 * (tr - 1.0);
    out3[3 * m + 1] = atan2(sn, cs) * (180.0 / 3.14159265358979323846);
    const double dx = Pg[3] - Pe[3], dy = Pg[7] - Pe[7], dz = Pg[11] - Pe[11];
    out3[3 * m + 2] = sqrt((dx * dx + dy * dy) + dz * dz);
  }
}
int pose_error2d_launch(const double *pose_est, const double *pose_gt, int M, const double *pts, int N, const double *K9,
                        double *out3, cudaStream_t st) {
  pose_error2d_kernel<<<M, 256, 0, st>>>(pose_est, pose_gt, pts, N, K9, out3);
  DIM_LAUNCH_CHECK();
  return 0;
}

int pose_error_launch(const double *pose_est, const double *pose_gt, int M, const double *pts, int N, int symmetric, double *out,
                      cudaStream_t st) {
  pose_error_kernel<<<M, 256, 0, st>>>(pose_est, pose_gt, pts, N, symmetric, out);
  DIM_LAUNCH_CHECK();
  return 0;
}

}  // namespace dim
