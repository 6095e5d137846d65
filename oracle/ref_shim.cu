// ref_shim.cu -- OUR C-ABI shim around the reference's CUDA voting launchers.
//
// TEST INFRASTRUCTURE ONLY (see oracle/pvnet_oracle.c header).  It is compiled by
// oracle/Makefile together with the reference project's lib/ransac_voting_gpu_layer/src/
// ransac_voting_kernel.cu -- taken verbatim from where it lies, never copied --
// into oracle/_ref/libpvnet_refcuda.so.  The reference's own binding
// (ransac_voting.cpp) does not compile against torch 2.11 (THCState, bare
// PYBIND11_MODULE), so this file stands in for it: raw device pointers in, the
// reference launchers called unchanged.
//
// Launchers declared here are defined at ransac_voting_kernel.cu:51-86 and
// :129-167 of the reference.
#include <ATen/ATen.h>
#include <cuda_runtime.h>
#include <cstdint>

at::Tensor generate_hypothesis_launcher(at::Tensor direct, at::Tensor coords, at::Tensor idxs);
void voting_for_hypothesis_launcher(at::Tensor direct, at::Tensor coords, at::Tensor hypo_pts,
                                    at::Tensor inliers, float inlier_thresh);

at::Tensor generate_hypothesis_vanishing_point_launcher(at::Tensor direct, at::Tensor coords, at::Tensor idxs);
void voting_for_hypothesis_vanishing_point_launcher(at::Tensor direct, at::Tensor coords, at::Tensor hypo_pts,
                                                    at::Tensor inliers, float inlier_thresh);

namespace {
at::Tensor wrap(void *p, at::IntArrayRef sizes, at::ScalarType t, int device)
{
    return at::from_blob(p, sizes, at::TensorOptions().dtype(t).device(at::kCUDA, device));
}
}  // namespace

extern "C" {

// direct [tn,vn,2] f32, coords [tn,2] f32, idxs [hn,vn,2] i32 -> hypo [hn,vn,2] f32.
// All device pointers on `device`; runs on the legacy default stream like the
// reference (ransac_voting_kernel.cu:76) and synchronises before returning.
__attribute__((visibility("default")))
int pvref_generate_hypothesis(float *direct, float *coords, int32_t *idxs, float *hypo_out,
                              int tn, int vn, int hn, int device)
{
    try {
        cudaSetDevice(device);
        at::Tensor d = wrap(direct, {tn, vn, 2}, at::kFloat, device);
        at::Tensor c = wrap(coords, {tn, 2}, at::kFloat, device);
        at::Tensor i = wrap(idxs, {hn, vn, 2}, at::kInt, device);
        at::Tensor h = generate_hypothesis_launcher(d, c, i);
        cudaError_t e = cudaMemcpy(hypo_out, h.data_ptr<float>(), sizeof(float) * (size_t)hn * vn * 2,
                                   cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) return (int)e;
        return (int)cudaDeviceSynchronize();
    } catch (...) {
        return -1;
    }
}

// inliers [hn,vn,tn] u8 must be zero-filled by the caller (ransac_voting_gpu.py:557).
__attribute__((visibility("default")))
int pvref_voting_for_hypothesis(float *direct, float *coords, float *hypo, uint8_t *inliers,
                                int tn, int vn, int hn, float thresh, int device)
{
    try {
        cudaSetDevice(device);
        at::Tensor d = wrap(direct, {tn, vn, 2}, at::kFloat, device);
        at::Tensor c = wrap(coords, {tn, 2}, at::kFloat, device);
        at::Tensor h = wrap(hypo, {hn, vn, 2}, at::kFloat, device);
        at::Tensor n = wrap(inliers, {hn, vn, tn}, at::kByte, device);
        voting_for_hypothesis_launcher(d, c, h, n, thresh);
        return (int)cudaDeviceSynchronize();
    } catch (...) {
        return -1;
    }
}

// the vanishing-point pair (ransac_voting_kernel.cu:232-260, :307-351): hypo [hn,vn,3]
__attribute__((visibility("default")))
int pvref_generate_hypothesis_vp(float *direct, float *coords, int32_t *idxs, float *hypo_out, int tn, int vn, int hn,
                                 int device)
{
    try {
        cudaSetDevice(device);
        at::Tensor h = generate_hypothesis_vanishing_point_launcher(wrap(direct, {tn, vn, 2}, at::kFloat, device),
                                                                    wrap(coords, {tn, 2}, at::kFloat, device),
                                                                    wrap(idxs, {hn, vn, 2}, at::kInt, device));
        cudaError_t e = cudaMemcpy(hypo_out, h.data_ptr<float>(), sizeof(float) * (size_t)hn * vn * 3,
                                   cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) return (int)e;
        return (int)cudaDeviceSynchronize();
    } catch (...) {
        return -1;
    }
}

__attribute__((visibility("default")))
int pvref_voting_for_hypothesis_vp(float *direct, float *coords, float *hypo, uint8_t *inliers, int tn, int vn, int hn,
                                   float thresh, int device)
{
    try {
        cudaSetDevice(device);
        voting_for_hypothesis_vanishing_point_launcher(wrap(direct, {tn, vn, 2}, at::kFloat, device),
                                                       wrap(coords, {tn, 2}, at::kFloat, device),
                                                       wrap(hypo, {hn, vn, 3}, at::kFloat, device),
                                                       wrap(inliers, {hn, vn, tn}, at::kByte, device), thresh);
        return (int)cudaDeviceSynchronize();
    } catch (...) {
        return -1;
    }
}

}  // extern "C"
