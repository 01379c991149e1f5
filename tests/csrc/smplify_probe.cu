// Test-only probe library (tests/libthmr_smplify_probe.so): extern "C" wrappers around the launchers of the fused
// SMPLify-inverse (tokenhmr_b200/csrc/smplify.cuh) that thmr_smplify_inv runs but the product ABI does not expose, so
// that tests/test_gpu_smplify_fused.py can check the loss / cotangent kernel against fp64 autograd and the Adam kernel
// against torch.optim.Adam one stage at a time.  The product never loads this library.
#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/smplify.cuh"

using namespace thmr;

#define PROBE_API extern "C" __attribute__((visibility("default")))

PROBE_API const char* smplify_probe_last_error(void) { return last_error_buf(); }

// smplify_loss_kernel as an iteration launches it (grad_joints / grad_cam non-null) or as the final forward does
// (both null, pj2d non-null); no done flag
PROBE_API int probe_smplify_loss(const float* joints, const float* cam, const float* focal, const float* kp2d,
                                 const float* kp3d, int J, int B, float* grad_joints, float* grad_cam, float* part,
                                 float* pj2d, void* stream) {
  return smplify_loss_launch(joints, cam, focal, kp2d, kp3d, J, B, grad_joints, grad_cam, part, pj2d, nullptr,
                             static_cast<cudaStream_t>(stream));
}

// smplify_adam_kernel for Adam step `step` (1-based) at learning rate lr over n flat elements; no done flag
PROBE_API int probe_smplify_adam(float* p, float* m, float* v, const float* g, long n, int step, double lr,
                                 void* stream) {
  return smplify_adam_launch(p, m, v, g, n, step, lr, nullptr, static_cast<cudaStream_t>(stream));
}
