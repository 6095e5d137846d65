// conv_tc.cuh -- internal interface of the tensor-core convolution (conv_tc.cu) and the
// auxiliary backbone kernels (backbone_aux.cu), shared with backbone.cu.
#pragma once
#include "common.cuh"

#include <cuda.h>
#ifdef __CUDACC__
#include "ptx.cuh"
#endif

namespace pvnet {

struct ConvDesc {
    const float *in;   // NHWC buffer [b,H,W,in_cs]; channels [in_co, in_co+Cin) are the conv input
    int in_cs, in_co, Cin;
    const float *w;    // packed [Cout][taps][Cin]
    const float *bias; // [Cout]
    const float *res;  // NHWC [b,Ho,Wo,res_cs] at res_co, or null
    int res_cs, res_co;
    float *out;        // NHWC [b,Ho,Wo,out_cs], written at out_co
    int out_cs, out_co, Cout;
    int b, H, W;
    int ksize, stride, dilation;
    int act, round_out;
    // optional second source (column kernel only): channels [Cin, Cin+Cin2) of the convolution come
    // from in2 [b,H,W,in2_cs] at in2_co -- a torch.cat on the READ side, so that both producers of a
    // concatenated input write dense records of their own
    const float *in2 = nullptr;
    int in2_cs = 0, in2_co = 0, Cin2 = 0;
};

// Optional fused 1x1 head (convraw.3 + argmax) for the column kernel's epilogue.
struct HeadDesc {
    const float *w;      // [cout][32] fp32
    const float *bias;   // [cout]
    float *out_nchw;     // [b,cout,H,W]
    void *mask;          // [b,H,W] int64 / u8, or null
    int mask_esz, seg_dim, cout;
};

// cuTensorMapEncodeTiled wrapper (fp32 elements); swizzle_bytes in {128,64,32}
int tma_encode(CUtensorMap *m, const void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides_bytes,
               const cuuint32_t *box, int swizzle_bytes);

// conv mode override for tests (pvnet_conv2d_nhwc only): 0 auto, 1 force per-tap kernel, 2 force column kernel
extern int g_conv_mode;
bool conv_col_eligible(const ConvDesc &d);
size_t conv_col_plan_size();
int conv_col_plan_at(const ConvDesc &d, const HeadDesc *head, void *plan_storage);
// The same for a two-source layer with Cin a multiple of 32, Cin2 == 8 and Cout 64 (Resnet50_8s_2o's conv2s.0): the
// first source in 32-channel chunks and the second as one more 8-channel chunk, instead of 8-channel chunks throughout.
int conv_col_plan_split_at(const ConvDesc &d, void *plan_storage);
int conv_col_launch_at(const void *plan_storage, cudaStream_t s);
void conv_col_set_head_ptrs(void *plan_storage, float *out, void *mask, int mask_esz, int nhwc);

// A plan = encoded tensor maps + launch geometry; opaque bytes so callers can cache it.
size_t conv_plan_size();
int conv_plan_at(const ConvDesc &d, void *plan_storage);
int conv_launch_at(const void *plan_storage, cudaStream_t s);

// half = 0: out is the full-resolution image slice [b,H,W,out_cs]; 1: x_ds [b,H/2,W/2,out_cs] (Resnet50_8s_2o);
// out = nullptr: s2d only (the detectors)
int launch_s2d_pack(const void *in, int in_is_u8, const float *mean3, const float *std3, float *s2d, float *out, int b,
                    int H, int W, int out_cs, int out_co, int half, cudaStream_t s);
int launch_maxpool(const float *in, float *out, int b, int H, int W, int C, int in_cs, int in_co, cudaStream_t s);
int launch_upsample2x(const float *in, float *out, int b, int h, int w, int C, int out_cs, int out_co,
                      cudaStream_t s);
// in NHWC [b,H,W,cin], cin 32 or 64 (raw_dim)
int launch_head(const float *in, int cin, const float *w, const float *bias, float *out, void *mask, int mask_esz,
                int seg_dim, int Cout, int b, int H, int W, int nhwc, cudaStream_t s);
// the detectors' 3x3 one-channel score head (head3x3.cu): in NHWC [b,H,W,C] dense, C a multiple of 32 up to 512,
// w [9][C], bias [1] -> out [b,1,H,W]
int launch_head3x3(const float *in, int C, const float *w, const float *bias, float *out, int b, int H, int W,
                   cudaStream_t s);

#ifdef __CUDACC__
// Three-slot interpolation sum with a FIXED rounding sequence (one weight of the window is zero): k_upsample2x
// goes through it, so its result does not depend on the contraction the compiler would have picked for
// `a*b + c*d + e*f`.
__device__ __forceinline__ float lerp3(float w0, float a, float w1, float b, float w2, float c)
{
    return __fmaf_rn(w2, c, __fmaf_rn(w1, b, __fmul_rn(w0, a)));
}
// Epilogue element shared by the conv kernels: activation, then optional rounding to tf32 (the value
// feeds another tensor-core conv).
__device__ __forceinline__ float epi_act(float v, int act, int round_out)
{
    if (act == 1) v = fmaxf(v, 0.f);
    else if (act == 2) v = fmaxf(v, 0.1f * v);       // LeakyReLU(0.1): max(x, 0.1x)
    return round_out ? ptx::round_tf32(v) : v;
}
#endif

}  // namespace pvnet
