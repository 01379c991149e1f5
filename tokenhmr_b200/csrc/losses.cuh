// TokenHMR's training / validation loss (thmr_tokenhmr_loss) and the differentiable camera tail (thmr_camera_tail,
// thmr_camera_tail_backward).
//
//   tokenhmr_loss_kernel   warp = sample: every per-sample term of TokenHMR.compute_loss (tokenhmr.py:190-277) and,
//                          when asked, the gradient of the weighted total w.r.t. the four predicted tensors.  Both
//                          branches: TALS (LOOSE_SUP and train, :214-249) and plain (:250-262).  The GT axis-angles go
//                          through geometry.aa_to_rotmat (quaternion route, +1e-8 in the norm), the angle test through
//                          rotation_utils.matrix_to_quaternion + quaternion_to_axis_angle, all in double, so every mask
//                          decision is the fp64 reference's.
//   tokenhmr_loss_reduce   one block: the batch sums of the five terms in a fixed order and the weighted total.
//
// Every loss of the reference is a sum over the batch, so a sample's gradient depends on that sample alone and is
// written by its own warp.  The masks carry no gradient; the L1 subgradient is sign (0 at 0), as torch's.  Nothing
// synchronises the host or allocates, and every sum has a fixed order: the call is bitwise reproducible and can be
// captured in a CUDA graph.  smpl_params_is_axis_angle is checked on the device: any sample whose flags are not the
// loaders' (True, True, False) raises g_loss_flags, which thmr_check_device_flags reports.
#pragma once
#include <cfloat>
#include <cmath>

#include "smpl_lbs.cuh"

namespace thmr {

__device__ unsigned int g_loss_flags = 0;   // set when a sample's smpl_params_is_axis_angle is unsupported

constexpr int kLossWarps = 4;            // samples per loss block
constexpr int kLossReduceThreads = 256;  // the batch reduction's single block
constexpr int kLossTerms = 5;            // per-sample sums: keypoints_2d, keypoints_3d, global_orient, body_pose, betas
constexpr int kLossTalsJoints = 44;      // entries of kp2D_err_valid_thresh

// losses.py:7-14 and :16-20, as the fp32 tensors the reference builds them; body_pose's is multiplied by 0.8 in fp32
__constant__ float c_kp2d_err_thresh[kLossTalsJoints] = {
    0.0085024f,  0.00648666f, 0.00747825f, 0.01103439f, 0.01355629f, 0.00741691f, 0.01096735f, 0.01414461f,
    0.00974212f, 0.01127469f, 0.01663222f, 0.00564927f, 0.01126335f, 0.01615757f, 0.00532595f, 0.00829731f,
    0.00831497f, 0.00737241f, 0.00743286f, 0.00543739f, 0.00550524f, 0.00535504f, 0.00565414f, 0.00581685f,
    0.00573041f, 0.00554029f, 0.01515258f, 0.00986267f, 0.00997563f, 0.01519944f, 0.00511402f, 0.01288267f,
    0.01105894f, 0.00710525f, 0.00709785f, 0.01092387f, 0.01388091f, 0.00648326f, 0.00766487f, 0.00931454f,
    0.00646622f, 0.00677057f, 0.00744011f, 0.00752381f};
__constant__ float c_body_angle_thresh[kSmplJ - 1] = {
    0.273709f,   0.26481161f, 0.1838198f,  0.41490657f, 0.37521194f, 0.20793171f, 0.24905021f, 0.33887333f,
    0.14481062f, 0.35632194f, 0.34944217f, 0.30542146f, 0.32835298f, 0.33110567f, 0.34813467f, 0.36357761f,
    0.40062272f, 0.43493496f, 0.4400709f,  0.78017052f, 0.7375746f,  0.24927082f, 0.24966981f};
constexpr float kGlobalOrientAngleThresh = 0.46f;

// geometry.py:5-44 aa_to_rotmat: the norm of theta + 1e-8, a unit quaternion, then quat_to_rotmat (row-major R)
__device__ __forceinline__ void aa_to_rotmat_quat(double x, double y, double z, double R[9]) {
  const double ex = x + 1e-8, ey = y + 1e-8, ez = z + 1e-8;
  const double n = sqrt(ex * ex + ey * ey + ez * ez);
  const double h = n * 0.5, c = cos(h), s = sin(h);
  double w = c, qx = s * (x / n), qy = s * (y / n), qz = s * (z / n);
  const double qn = sqrt(w * w + qx * qx + qy * qy + qz * qz);
  w /= qn; qx /= qn; qy /= qn; qz /= qn;
  const double w2 = w * w, x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
  const double wx = w * qx, wy = w * qy, wz = w * qz, xy = qx * qy, xz = qx * qz, yz = qy * qz;
  R[0] = w2 + x2 - y2 - z2; R[1] = 2 * xy - 2 * wz;     R[2] = 2 * wy + 2 * xz;
  R[3] = 2 * wz + 2 * xy;   R[4] = w2 - x2 + y2 - z2;   R[5] = 2 * yz - 2 * wx;
  R[6] = 2 * xz - 2 * wy;   R[7] = 2 * wx + 2 * yz;     R[8] = w2 - x2 - y2 + z2;
}

// |matrix_to_axis_angle(m)|: rotation_utils.matrix_to_quaternion (the best-conditioned of the four candidates, no
// standardisation, rotation_utils.py:104-163) then quaternion_to_axis_angle (:478-506), in the same steps
__device__ __forceinline__ double rotation_angle(const double m[9]) {
  const double t[4] = {1.0 + m[0] + m[4] + m[8], 1.0 + m[0] - m[4] - m[8], 1.0 - m[0] + m[4] - m[8],
                       1.0 - m[0] - m[4] + m[8]};
  int k = 0;
  double qk = 0.0;   // q_abs[argmax], the first maximum
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double q = t[i] > 0.0 ? sqrt(t[i]) : 0.0;
    if (i == 0 || q > qk) { k = i; qk = q; }
  }
  double r[4];
  if (k == 0) { r[0] = qk * qk; r[1] = m[7] - m[5]; r[2] = m[2] - m[6]; r[3] = m[3] - m[1]; }
  else if (k == 1) { r[0] = m[7] - m[5]; r[1] = qk * qk; r[2] = m[3] + m[1]; r[3] = m[2] + m[6]; }
  else if (k == 2) { r[0] = m[2] - m[6]; r[1] = m[3] + m[1]; r[2] = qk * qk; r[3] = m[5] + m[7]; }
  else { r[0] = m[3] - m[1]; r[1] = m[6] + m[2]; r[2] = m[7] + m[5]; r[3] = qk * qk; }
  const double den = fmax(2.0 * fmax(qk, 0.1), DBL_MIN);
  const double q0 = r[0] / den, q1 = r[1] / den, q2 = r[2] / den, q3 = r[3] / den;
  const double half = atan2(sqrt(q1 * q1 + q2 * q2 + q3 * q3), q0), ang = 2.0 * half;
  double s = fabs(ang) < 1e-6 ? 0.5 - ang * ang / 48.0 : sin(half) / ang;
  s = fmax(s, DBL_MIN);
  const double a1 = q1 / s, a2 = q2 / s, a3 = q3 / s;
  return sqrt(a1 * a1 + a2 * a2 + a3 * a3);
}

__device__ __forceinline__ double sgn(double x) { return x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : 0.0); }

__device__ __forceinline__ double warp_sum(double v) {
  // butterfly: every lane ends with the same, fixed-order sum
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// part [B,kLossTerms] <- per-sample sums of the five terms (each already in its branch's masking, unweighted).
// The four gradients (all set or all null) are those of the weighted total, for a unit upstream gradient.
__global__ void __launch_bounds__(32 * kLossWarps)
tokenhmr_loss_kernel(const thmr_loss_desc d, double* __restrict__ part) {
  const int b = blockIdx.x * kLossWarps + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (b >= d.B) return;
  const int J = d.num_joints, nb = d.num_betas, pel = d.pelvis_id;
  const bool tals = d.tals != 0, grads = d.grad_keypoints_2d != nullptr;
  const double lw = d.loose_weight;
  if (lane == 0 && !(d.is_axis_angle_global_orient[b] && d.is_axis_angle_body_pose[b] && !d.is_axis_angle_betas[b]))
    atomicExch(&g_loss_flags, 1u);
  const double v3d = tals ? static_cast<double>(d.valid_3d[b]) : 0.0;

  // ---- keypoints: 2-D L1 (TALS: full weight above the per-joint threshold, LOOSE_WEIGHT below) and the
  //      pelvis-aligned 3-D L1 (TALS: gated by valid_3D + the masked 2-D confidence)
  const size_t kb = static_cast<size_t>(b) * J;
  const float* p2 = d.pred_keypoints_2d + kb * 2;
  const float* g2 = d.gt_keypoints_2d + kb * 3;
  const float* p3 = d.pred_keypoints_3d + kb * 3;
  const float* g3 = d.gt_keypoints_3d + kb * 4;
  const double pp[3] = {p3[pel * 3 + 0], p3[pel * 3 + 1], p3[pel * 3 + 2]};
  const double gp[3] = {g3[pel * 4 + 0], g3[pel * 4 + 1], g3[pel * 4 + 2]};
  double s2 = 0.0, s3 = 0.0, gpel[3] = {0.0, 0.0, 0.0};
  for (int j = lane; j < J; j += 32) {
    const double c = g2[j * 3 + 2];
    const double dx = static_cast<double>(p2[j * 2 + 0]) - g2[j * 3 + 0];
    const double dy = static_cast<double>(p2[j * 2 + 1]) - g2[j * 3 + 1];
    double w2 = c, cm = c;
    if (tals) {
      const bool valid = c * (dx * dx + dy * dy) > static_cast<double>(c_kp2d_err_thresh[j]);
      cm = c * (valid ? 1.0 : 0.0);                         // gt_keypoints_2d[:, :, -1] after tokenhmr.py:223
      w2 = valid ? c : lw * (c * 1.0);                      // conf + LOOSE_WEIGHT * weak_mask
    }
    s2 += w2 * (fabs(dx) + fabs(dy));
    double c3 = g3[j * 4 + 3];
    if (tals) c3 *= (v3d + cm) > 0.5 ? 1.0 : 0.0;
    double e3[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
      e3[i] = (static_cast<double>(p3[j * 3 + i]) - pp[i]) - (static_cast<double>(g3[j * 4 + i]) - gp[i]);
    s3 += c3 * (fabs(e3[0]) + fabs(e3[1]) + fabs(e3[2]));
    if (grads) {
      const double a2 = d.w_keypoints_2d * w2, a3 = d.w_keypoints_3d * c3;
      d.grad_keypoints_2d[(kb + j) * 2 + 0] = static_cast<float>(a2 * sgn(dx));
      d.grad_keypoints_2d[(kb + j) * 2 + 1] = static_cast<float>(a2 * sgn(dy));
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double g = a3 * sgn(e3[i]);
        gpel[i] -= g;
        if (j != pel) d.grad_keypoints_3d[(kb + j) * 3 + i] = static_cast<float>(g);
      }
    }
  }

  // ---- rotations (lane k < 24: global_orient, then body_pose[k-1]) against the GT axis-angles
  double sgo = 0.0, sbp = 0.0, sbe = 0.0;
  if (lane < kSmplJ) {
    const int k = lane;
    const float* aa = k == 0 ? d.gt_global_orient + b * 3 : d.gt_body_pose + static_cast<size_t>(b) * 69 + (k - 1) * 3;
    double G[9], P[9];
    aa_to_rotmat_quat(aa[0], aa[1], aa[2], G);
    const float* R = d.pred_rotmats + (static_cast<size_t>(b) * kSmplJ + k) * 9;
    double e = 0.0;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      P[i] = R[i];
      e += (P[i] - G[i]) * (P[i] - G[i]);
    }
    const double has = k == 0 ? d.has_global_orient[b] : d.has_body_pose[b];
    double w = has;
    if (tals) {
      double r[9];   // R_pred R_gt^T
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int c = 0; c < 3; ++c) r[i * 3 + c] = P[i * 3] * G[c * 3] + P[i * 3 + 1] * G[c * 3 + 1] + P[i * 3 + 2] * G[c * 3 + 2];
      const float thr = k == 0 ? kGlobalOrientAngleThresh : __fmul_rn(c_body_angle_thresh[k - 1], 0.8f);
      const bool valid = rotation_angle(r) > static_cast<double>(thr);
      // valid_mask3D = (valid * has + valid_3D).bool(); weak = ~valid_mask3D * has  (tokenhmr.py:244-247)
      const bool mask = ((valid ? 1.0 : 0.0) * has + v3d) != 0.0;
      w = mask ? 1.0 : lw * has;
    }
    (k == 0 ? sgo : sbp) = w * e;
    if (grads) {
      const double a = 2.0 * w * (k == 0 ? d.w_global_orient : d.w_body_pose);
      float* gr = d.grad_rotmats + (static_cast<size_t>(b) * kSmplJ + k) * 9;
#pragma unroll
      for (int i = 0; i < 9; ++i) gr[i] = static_cast<float>(a * (P[i] - G[i]));
    }
  }
  // ---- betas: has (TALS: has * valid_3D) times the squared error
  const double hb = static_cast<double>(d.has_betas[b]) * (tals ? v3d : 1.0);
  for (int i = lane; i < nb; i += 32) {
    const size_t o = static_cast<size_t>(b) * nb + i;
    const double e = static_cast<double>(d.pred_betas[o]) - d.gt_betas[o];
    sbe += hb * (e * e);
    if (grads) d.grad_betas[o] = static_cast<float>(2.0 * hb * d.w_betas * e);
  }

  s2 = warp_sum(s2); s3 = warp_sum(s3); sgo = warp_sum(sgo); sbp = warp_sum(sbp); sbe = warp_sum(sbe);
  if (grads) {
#pragma unroll
    for (int i = 0; i < 3; ++i) gpel[i] = warp_sum(gpel[i]);
  }
  if (lane == 0) {
    double* o = part + static_cast<size_t>(b) * kLossTerms;
    o[0] = s2; o[1] = s3; o[2] = sgo; o[3] = sbp; o[4] = sbe;
    if (grads)
      for (int i = 0; i < 3; ++i) d.grad_keypoints_3d[(kb + pel) * 3 + i] = static_cast<float>(gpel[i]);
  }
}

// losses [6] <- (loss, keypoints_2d, keypoints_3d, global_orient, body_pose, betas): batch sums in a fixed order,
// then loss = w3d l3d + w2d l2d + (l_go w_go + l_bp w_bp + l_betas w_betas) as tokenhmr.py:264-266 adds them
__global__ void __launch_bounds__(kLossReduceThreads)
tokenhmr_loss_reduce(const double* __restrict__ part, int B, const thmr_loss_desc d) {
  __shared__ double s[kLossTerms][kLossReduceThreads];
  const int t = threadIdx.x;
  double a[kLossTerms] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = t; b < B; b += kLossReduceThreads)
#pragma unroll
    for (int i = 0; i < kLossTerms; ++i) a[i] += part[static_cast<size_t>(b) * kLossTerms + i];
#pragma unroll
  for (int i = 0; i < kLossTerms; ++i) s[i][t] = a[i];
  __syncthreads();
  for (int w = kLossReduceThreads / 2; w > 0; w >>= 1) {
    if (t < w)
#pragma unroll
      for (int i = 0; i < kLossTerms; ++i) s[i][t] += s[i][t + w];
    __syncthreads();
  }
  if (t != 0) return;
  const double l2 = s[0][0], l3 = s[1][0], lgo = s[2][0], lbp = s[3][0], lbe = s[4][0];
  const double loss = d.w_keypoints_3d * l3 + d.w_keypoints_2d * l2 + (lgo * d.w_global_orient + lbp * d.w_body_pose +
                                                                       lbe * d.w_betas);
  d.losses[0] = static_cast<float>(loss);
  d.losses[1] = static_cast<float>(l2);
  d.losses[2] = static_cast<float>(l3);
  d.losses[3] = static_cast<float>(lgo);
  d.losses[4] = static_cast<float>(lbp);
  d.losses[5] = static_cast<float>(lbe);
}

inline size_t tokenhmr_loss_part_bytes(int B) { return static_cast<size_t>(B) * kLossTerms * sizeof(double); }

inline int tokenhmr_loss_run(const thmr_loss_desc& d, void* workspace, cudaStream_t st) {
  double* part = static_cast<double*>(workspace);
  tokenhmr_loss_kernel<<<(d.B + kLossWarps - 1) / kLossWarps, 32 * kLossWarps, 0, st>>>(d, part);
  THMR_CUDA(cudaGetLastError());
  tokenhmr_loss_reduce<<<1, kLossReduceThreads, 0, st>>>(part, d.B, d);
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

// ---- camera tail --------------------------------------------------------------------------------------------------
constexpr int kTailWarps = 4;   // samples per camera-tail block (one warp each)

// joints [B,J,3], pred_cam [B,3] -> cam_t [B,3], focal_out [B,2] (nullable), kp2d [B,J,2]; the numbers
// smpl_joints_kernel writes for the same joints and camera (the same two expressions)
__global__ void __launch_bounds__(32 * kTailWarps)
camera_tail_kernel(const float* __restrict__ joints, const float* __restrict__ pred_cam, int J, int B, float focal,
                   float image_size, float* __restrict__ cam_t, float* __restrict__ focal_out,
                   float* __restrict__ kp2d) {
  const int b = blockIdx.x * kTailWarps + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (b >= B) return;
  const float t[3] = {pred_cam[b * 3 + 1], pred_cam[b * 3 + 2], cam_depth(pred_cam[b * 3 + 0], focal, image_size)};
  if (lane == 0) {
    cam_t[b * 3 + 0] = t[0]; cam_t[b * 3 + 1] = t[1]; cam_t[b * 3 + 2] = t[2];
    if (focal_out) { focal_out[b * 2 + 0] = focal; focal_out[b * 2 + 1] = focal; }
  }
  for (int j = lane; j < J; j += 32) {
    const size_t r = static_cast<size_t>(b) * J + j;
    const float x[3] = {joints[r * 3 + 0], joints[r * 3 + 1], joints[r * 3 + 2]};
    const float2 u = project_point(x, t, focal, image_size);
    kp2d[r * 2 + 0] = u.x;
    kp2d[r * 2 + 1] = u.y;
  }
}

// VJP of camera_tail_kernel: grad_kp2d [B,J,2] and grad_cam_t [B,3] (each nullable = zero) -> grad_joints [B,J,3] and
// grad_pred_cam [B,3].  Stateless: the forward's values are recomputed from joints and pred_cam.
__global__ void __launch_bounds__(32 * kTailWarps)
camera_tail_backward_kernel(const float* __restrict__ joints, const float* __restrict__ pred_cam, int J, int B,
                            float focal, float image_size, const float* __restrict__ grad_kp2d,
                            const float* __restrict__ grad_cam_t, float* __restrict__ grad_joints,
                            float* __restrict__ grad_pred_cam) {
  const int b = blockIdx.x * kTailWarps + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (b >= B) return;
  const float s = pred_cam[b * 3 + 0];
  const float t[3] = {pred_cam[b * 3 + 1], pred_cam[b * 3 + 2], cam_depth(s, focal, image_size)};
  const float f = focal / image_size;
  float gx = 0.f, gy = 0.f, gz = 0.f;
  for (int j = lane; j < J; j += 32) {
    const size_t r = static_cast<size_t>(b) * J + j;
    const float px = joints[r * 3 + 0] + t[0], py = joints[r * 3 + 1] + t[1], pz = joints[r * 3 + 2] + t[2];
    float gpx = 0.f, gpy = 0.f, gpz = 0.f;
    if (grad_kp2d) {
      // u = f q, q = p_xy / p_z
      const float gqx = f * grad_kp2d[r * 2 + 0], gqy = f * grad_kp2d[r * 2 + 1];
      gpx = gqx / pz;
      gpy = gqy / pz;
      gpz = -(gqx * (px / pz) + gqy * (py / pz)) / pz;
    }
    grad_joints[r * 3 + 0] = gpx; grad_joints[r * 3 + 1] = gpy; grad_joints[r * 3 + 2] = gpz;
    gx += gpx; gy += gpy; gz += gpz;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gx += __shfl_xor_sync(0xffffffffu, gx, o);
    gy += __shfl_xor_sync(0xffffffffu, gy, o);
    gz += __shfl_xor_sync(0xffffffffu, gz, o);
  }
  if (lane != 0) return;
  if (grad_cam_t) { gx += grad_cam_t[b * 3 + 0]; gy += grad_cam_t[b * 3 + 1]; gz += grad_cam_t[b * 3 + 2]; }
  // t_z = 2 focal / (image_size s + 1e-9):  d t_z / d s = -2 focal image_size / (image_size s + 1e-9)^2
  const float den = image_size * s + 1e-9f;
  grad_pred_cam[b * 3 + 0] = gz * (-2.f * focal * image_size / (den * den));
  grad_pred_cam[b * 3 + 1] = gx;
  grad_pred_cam[b * 3 + 2] = gy;
}

}  // namespace thmr
