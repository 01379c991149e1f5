// SMPLify-inverse as one stream-ordered call (thmr_smplify_inv): the loop body of smplify_invert.py:114-132 for every
// sample of the batch, then the final forward of :135-149.  One iteration is
//
//   smpl_run               the body model's forward on the packed rotations [B,24,3,3] (no camera tail): joints
//   smplify_loss_kernel    warp = sample: projection at focal / 256, the per-sample fit2D and push3D sums, and the
//                          cotangents of loss = 4 mean(fit2D) - mean(push3D) / 2 + margin w.r.t. the joints and pred_cam_t
//   smplify_reduce_kernel  one block: batch means, the loss in the reference's fp32 operation order, the history row and
//                          the stop test (in double, as the reference compares .item() values with Python floats)
//   smpl_backward_run      the body model's backward with the joint cotangent only
//   smplify_adam_kernel    torch.optim.Adam's step (torch 2.11 _multi_tensor_adam, non-capturable branch) on
//                          [rotations | pred_cam_t] as one flat array
//
// Once the stop test fires, the loss, reduce and Adam kernels of every later iteration return at once; the forward and
// backward still run on the unchanged parameters (wasted time after an early stop, never a change of result).  Every
// reduction runs in a fixed order without atomics, and nothing synchronises the host or allocates, so the call is
// bitwise reproducible and can be captured in a CUDA graph.
#pragma once
#include <cmath>

#include "smpl_grad.cuh"

namespace thmr {

constexpr int kFitWarps = 4;              // samples per loss block (one warp each)
constexpr int kFitReduceThreads = 256;    // the batch reduction's single block
constexpr int kFitRot = kSmplJ * 9;       // packed rotation floats per sample

// Workspace of thmr_smplify_inv, carved by smplify_carve.
struct SmplifyWs {
  SmplBwdWs bwd;     // the body model's forward (bwd.fwd) and backward workspaces
  float* verts;      // [B,V,3]    vertices of the iteration forwards (not returned)
  float* param;      // [B*216 + B*3]  packed global_orient | body_pose per sample, then pred_cam_t
  float* exp_avg;    // Adam first moment, param's layout
  float* exp_avg_sq; // Adam second moment, param's layout
  float* grad;       // loss gradient, param's layout: rotations from the backward, pred_cam_t from the loss kernel
  float* grad_betas; // [B,nb]     written by the backward, unused (betas are not optimised)
  float* joints;     // [B,J,3]
  float* grad_joints;// [B,J,3]    joint cotangent
  float* part;       // [2,B]      per-sample fit2D, push3D
  float* history;    // [max(num_iters,1),3]  (loss, fit2D, mean push3D) per iteration run; zero past the stop
  int* state;        // [2]        done flag, iterations run
};

inline void smplify_carve(Bump& bp, const SmplModel& m, int B, int num_iters, SmplifyWs* ws) {
  smpl_bwd_carve(bp, m, B, &ws->bwd);
  const size_t b = static_cast<size_t>(B), J = static_cast<size_t>(25 + m.n_extra);
  const size_t np = b * (kFitRot + 3);
  ws->verts = bp.take<float>(b * m.V * 3);
  ws->param = bp.take<float>(np);
  ws->exp_avg = bp.take<float>(np);
  ws->exp_avg_sq = bp.take<float>(np);
  ws->grad = bp.take<float>(np);
  ws->grad_betas = bp.take<float>(b * m.nb);
  ws->joints = bp.take<float>(b * J * 3);
  ws->grad_joints = bp.take<float>(b * J * 3);
  ws->part = bp.take<float>(2 * b);
  ws->history = bp.take<float>(static_cast<size_t>(num_iters > 0 ? num_iters : 1) * 3);
  ws->state = bp.take<int>(2);
}

// ---- per-sample loss terms and cotangents ------------------------------------------------------------------------
//   joints [B,J,3], cam [B,3], focal [B,2], kp2d [B,J,3] (confidence column unused), kp3d [B,J,3]
//   part [2,B] <- per-sample sum_j |kp2d - proj| and sum_j |joints - kp3d|
//   grad_joints [B,J,3] and grad_cam [B,3] (both nullable together): the cotangents of the loss, whose 1/B factors are
//   the constants 4/B and -0.5/B.  The sqrt backward is torch's g / (2 sqrt(s)) times 2r, so a residual of exactly
//   zero gives autograd's NaN.
//   pj2d [B,J,2] (nullable) <- the projected joints
//   state (nullable): the kernel returns at once when state[0] (done) is set
__global__ void __launch_bounds__(32 * kFitWarps)
smplify_loss_kernel(const float* __restrict__ joints, const float* __restrict__ cam, const float* __restrict__ focal,
                    const float* __restrict__ kp2d, const float* __restrict__ kp3d, int J, int B,
                    float* __restrict__ grad_joints, float* __restrict__ grad_cam, float* __restrict__ part,
                    float* __restrict__ pj2d, const int* __restrict__ state) {
  if (state && state[0]) return;
  const int b = blockIdx.x * kFitWarps + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (b >= B) return;
  const float tx = cam[b * 3 + 0], ty = cam[b * 3 + 1], tz = cam[b * 3 + 2];
  const float cx = __fdiv_rn(focal[b * 2 + 0], 256.f), cy = __fdiv_rn(focal[b * 2 + 1], 256.f);
  const float g2 = __fdiv_rn(4.f, static_cast<float>(B));     // d loss / d |r2d|
  const float g3 = __fdiv_rn(-0.5f, static_cast<float>(B));   // d loss / d |r3d|
  float f2 = 0.f, f3 = 0.f, gcx = 0.f, gcy = 0.f, gcz = 0.f;
  for (int j = lane; j < J; j += 32) {
    const size_t r = static_cast<size_t>(b) * J + j;
    const float jx = joints[r * 3 + 0], jy = joints[r * 3 + 1], jz = joints[r * 3 + 2];
    const float px = __fadd_rn(jx, tx), py = __fadd_rn(jy, ty), pz = __fadd_rn(jz, tz);
    const float qx = __fdiv_rn(px, pz), qy = __fdiv_rn(py, pz);
    const float ux = __fmul_rn(cx, qx), uy = __fmul_rn(cy, qy);
    const float dx = __fsub_rn(kp2d[r * 3 + 0], ux), dy = __fsub_rn(kp2d[r * 3 + 1], uy);
    const float r2 = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    const float ex = __fsub_rn(jx, kp3d[r * 3 + 0]), ey = __fsub_rn(jy, kp3d[r * 3 + 1]);
    const float ez = __fsub_rn(jz, kp3d[r * 3 + 2]);
    const float r3 = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)));
    f2 = __fadd_rn(f2, r2);
    f3 = __fadd_rn(f3, r3);
    if (pj2d) { pj2d[r * 2 + 0] = ux; pj2d[r * 2 + 1] = uy; }
    if (grad_joints) {
      const float h2 = __fdiv_rn(g2, __fmul_rn(2.f, r2)), h3 = __fdiv_rn(g3, __fmul_rn(2.f, r3));
      // d = kp - u:  u_bar = -h2 * 2d;  u = c q:  q_bar = c u_bar;  q = p_xy / p_z
      const float gqx = __fmul_rn(cx, -__fmul_rn(h2, __fmul_rn(2.f, dx)));
      const float gqy = __fmul_rn(cy, -__fmul_rn(h2, __fmul_rn(2.f, dy)));
      const float gpx = __fdiv_rn(gqx, pz), gpy = __fdiv_rn(gqy, pz);
      const float gpz = -__fdiv_rn(__fadd_rn(__fmul_rn(gqx, qx), __fmul_rn(gqy, qy)), pz);
      grad_joints[r * 3 + 0] = __fadd_rn(gpx, __fmul_rn(h3, __fmul_rn(2.f, ex)));
      grad_joints[r * 3 + 1] = __fadd_rn(gpy, __fmul_rn(h3, __fmul_rn(2.f, ey)));
      grad_joints[r * 3 + 2] = __fadd_rn(gpz, __fmul_rn(h3, __fmul_rn(2.f, ez)));
      gcx = __fadd_rn(gcx, gpx); gcy = __fadd_rn(gcy, gpy); gcz = __fadd_rn(gcz, gpz);
    }
  }
  // butterfly: every lane ends with the same, fixed-order sums (each step adds the same pair in either order)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f2 = __fadd_rn(f2, __shfl_xor_sync(0xffffffffu, f2, o));
    f3 = __fadd_rn(f3, __shfl_xor_sync(0xffffffffu, f3, o));
    gcx = __fadd_rn(gcx, __shfl_xor_sync(0xffffffffu, gcx, o));
    gcy = __fadd_rn(gcy, __shfl_xor_sync(0xffffffffu, gcy, o));
    gcz = __fadd_rn(gcz, __shfl_xor_sync(0xffffffffu, gcz, o));
  }
  if (lane == 0) {
    part[b] = f2;
    part[B + b] = f3;
    if (grad_cam) { grad_cam[b * 3 + 0] = gcx; grad_cam[b * 3 + 1] = gcy; grad_cam[b * 3 + 2] = gcz; }
  }
}

// ---- batch means, loss, history and stop test (single block) -----------------------------------------------------
//   iteration mode (reproj == nullptr): history[it] <- (loss, fit2D, mean push3D), state[1] <- it + 1, and state[0] <- 1
//   when loss < thr_f3d and fit2D < thr_f2d; returns at once when state[0] is already set.
//   final mode: *reproj <- mean fit2D (camera_fitting_loss).
__global__ void __launch_bounds__(kFitReduceThreads)
smplify_reduce_kernel(const float* __restrict__ part, int B, float margin, double thr_f2d, double thr_f3d, int it,
                      float* __restrict__ history, int* __restrict__ state, float* __restrict__ reproj) {
  if (!reproj && state[0]) return;
  __shared__ float s2[kFitReduceThreads], s3[kFitReduceThreads];
  const int t = threadIdx.x;
  float a = 0.f, c = 0.f;
  for (int b = t; b < B; b += kFitReduceThreads) { a = __fadd_rn(a, part[b]); c = __fadd_rn(c, part[B + b]); }
  s2[t] = a;
  s3[t] = c;
  __syncthreads();
  for (int w = kFitReduceThreads / 2; w > 0; w >>= 1) {
    if (t < w) { s2[t] = __fadd_rn(s2[t], s2[t + w]); s3[t] = __fadd_rn(s3[t], s3[t + w]); }
    __syncthreads();
  }
  if (t != 0) return;
  const float fit = __fdiv_rn(s2[0], static_cast<float>(B)), push = __fdiv_rn(s3[0], static_cast<float>(B));
  if (reproj) { *reproj = fit; return; }
  // smplify_invert.py:124  loss = 4*fit2D - push3D.mean() /2 + self.margin
  const float loss = __fadd_rn(__fsub_rn(__fmul_rn(4.f, fit), __fdiv_rn(push, 2.f)), margin);
  history[it * 3 + 0] = loss;
  history[it * 3 + 1] = fit;
  history[it * 3 + 2] = push;
  state[1] = it + 1;
  if (static_cast<double>(loss) < thr_f3d && static_cast<double>(fit) < thr_f2d) state[0] = 1;
}

// ---- Adam ----------------------------------------------------------------------------------------------------------
// The float scalars torch's foreach kernels receive for one step (betas (0.9, 0.999), eps 1e-8, no weight decay):
// the bias corrections are Python floats (double) converted to float at the kernel boundary.
struct AdamScalars {
  float w1;         // lerp weight 1 - beta1
  float beta2;
  float w2;         // addcmul value 1 - beta2
  float bc2_sqrt;   // (1 - beta2^step) ** 0.5
  float eps;
  float step_size;  // (lr / (1 - beta1^step)) * -1
};
inline AdamScalars adam_scalars(int step, double lr) {
  const double beta1 = 0.9, beta2 = 0.999;
  const double bc1 = 1.0 - std::pow(beta1, static_cast<double>(step));
  const double bc2 = 1.0 - std::pow(beta2, static_cast<double>(step));
  AdamScalars s;
  s.w1 = static_cast<float>(1.0 - beta1);
  s.beta2 = static_cast<float>(beta2);
  s.w2 = static_cast<float>(1.0 - beta2);
  s.bc2_sqrt = static_cast<float>(std::pow(bc2, 0.5));
  s.eps = static_cast<float>(1e-8);
  s.step_size = static_cast<float>((lr / bc1) * -1.0);
  return s;
}

// One element per thread, each operation rounded where torch's kernel rounds it:
//   _foreach_lerp_(m, g, w1)        m + w1 (g - m)          (weight < 0.5 branch of at::native::lerp; fused)
//   _foreach_mul_(v, beta2)         v beta2
//   _foreach_addcmul_(v, g, g, w2)  v + w2 (g g)            (fused)
//   _foreach_sqrt / _foreach_div_(bc2_sqrt) / _foreach_add_(eps)
//   _foreach_addcdiv_(p, m, d, s)   p + s (m / d)           (fused)
__global__ void __launch_bounds__(256)
smplify_adam_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v, const float* __restrict__ g,
                    long n, AdamScalars s, const int* __restrict__ state) {
  if (state && state[0]) return;
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  const float mi = __fmaf_rn(s.w1, __fsub_rn(gi, m[i]), m[i]);
  const float vi = __fmaf_rn(s.w2, __fmul_rn(gi, gi), __fmul_rn(v[i], s.beta2));
  const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), s.bc2_sqrt), s.eps);
  p[i] = __fmaf_rn(s.step_size, __fdiv_rn(mi, d), p[i]);
  m[i] = mi;
  v[i] = vi;
}

inline int smplify_adam_launch(float* p, float* m, float* v, const float* g, long n, int step, double lr,
                               const int* state, cudaStream_t st) {
  smplify_adam_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(p, m, v, g, n, adam_scalars(step, lr),
                                                                               state);
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

inline int smplify_loss_launch(const float* joints, const float* cam, const float* focal, const float* kp2d,
                               const float* kp3d, int J, int B, float* grad_joints, float* grad_cam, float* part,
                               float* pj2d, const int* state, cudaStream_t st) {
  smplify_loss_kernel<<<(B + kFitWarps - 1) / kFitWarps, 32 * kFitWarps, 0, st>>>(
      joints, cam, focal, kp2d, kp3d, J, B, grad_joints, grad_cam, part, pj2d, state);
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

// The whole fit.  d has been validated (thmr_smplify_inv); ws carved for (d.B, d.num_iters).
inline int smplify_run(const thmr_smpl* sm, const thmr_smplify_desc& d, const SmplifyWs& ws, cudaStream_t st) {
  const int B = d.B, J = d.num_joints;
  const size_t nrot = static_cast<size_t>(B) * kFitRot, np = nrot + static_cast<size_t>(B) * 3;
  float* cam = ws.param + nrot;
  const size_t F = sizeof(float);
  // pack the parameters, zero the Adam state, the history and the done flag / count
  THMR_CUDA(cudaMemcpy2DAsync(ws.param, kFitRot * F, d.global_orient, 9 * F, 9 * F, B, cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemcpy2DAsync(ws.param + 9, kFitRot * F, d.body_pose, 23 * 9 * F, 23 * 9 * F, B,
                              cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemcpyAsync(cam, d.pred_cam_t, static_cast<size_t>(B) * 3 * F, cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemsetAsync(ws.exp_avg, 0, np * F, st));
  THMR_CUDA(cudaMemsetAsync(ws.exp_avg_sq, 0, np * F, st));
  THMR_CUDA(cudaMemsetAsync(ws.history, 0, static_cast<size_t>(d.num_iters > 0 ? d.num_iters : 1) * 3 * F, st));
  THMR_CUDA(cudaMemsetAsync(ws.state, 0, 2 * sizeof(int), st));
  const float margin = static_cast<float>(d.margin);
  for (int it = 0; it < d.num_iters; ++it) {
    THMR_TRY(smpl_run(sm, ws.param, 0, d.betas, B, ws.verts, nullptr, ws.joints, nullptr, 0.f, 0.f, nullptr, nullptr,
                      nullptr, ws.bwd.fwd, nullptr, st));
    THMR_TRY(smplify_loss_launch(ws.joints, cam, d.focal_length, d.gt_keypoints_2d, d.gt_keypoints_3d, J, B,
                                 ws.grad_joints, ws.grad + nrot, ws.part, nullptr, ws.state, st));
    smplify_reduce_kernel<<<1, kFitReduceThreads, 0, st>>>(ws.part, B, margin, d.loss_thresh_f2d, d.loss_thresh_f3d,
                                                           it, ws.history, ws.state, nullptr);
    THMR_CUDA(cudaGetLastError());
    THMR_TRY(smpl_backward_run(sm, ws.param, 0, d.betas, B, nullptr, ws.grad_joints, 0, ws.grad, ws.grad_betas, ws.bwd,
                               st));
    // the step count of every parameter is it + 1: no step follows a stop
    THMR_TRY(smplify_adam_launch(ws.param, ws.exp_avg, ws.exp_avg_sq, ws.grad, static_cast<long>(np), it + 1,
                                 d.step_size, ws.state, st));
  }
  // final forward on the final parameters (smplify_invert.py:135-149)
  THMR_TRY(smpl_run(sm, ws.param, 0, d.betas, B, d.vertices, nullptr, d.joints, nullptr, 0.f, 0.f, nullptr, nullptr,
                    nullptr, ws.bwd.fwd, nullptr, st));
  THMR_TRY(smplify_loss_launch(d.joints, cam, d.focal_length, d.gt_keypoints_2d, d.gt_keypoints_3d, J, B, nullptr,
                               nullptr, ws.part, d.pj2ds, nullptr, st));
  smplify_reduce_kernel<<<1, kFitReduceThreads, 0, st>>>(ws.part, B, margin, 0.0, 0.0, 0, nullptr, nullptr,
                                                         d.reprojection_loss);
  THMR_CUDA(cudaGetLastError());
  // the caller's parameters, history and iteration count
  THMR_CUDA(cudaMemcpy2DAsync(d.global_orient, 9 * F, ws.param, kFitRot * F, 9 * F, B, cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemcpy2DAsync(d.body_pose, 23 * 9 * F, ws.param + 9, kFitRot * F, 23 * 9 * F, B,
                              cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemcpyAsync(d.pred_cam_t, cam, static_cast<size_t>(B) * 3 * F, cudaMemcpyDeviceToDevice, st));
  if (d.num_iters > 0)
    THMR_CUDA(cudaMemcpyAsync(d.history, ws.history, static_cast<size_t>(d.num_iters) * 3 * F,
                              cudaMemcpyDeviceToDevice, st));
  THMR_CUDA(cudaMemcpyAsync(d.iters_run, ws.state + 1, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return THMR_OK;
}

}  // namespace thmr
