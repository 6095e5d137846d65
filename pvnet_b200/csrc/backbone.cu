// backbone.cu -- Resnet18_8s.forward (lib/networks/model_repository.py:64-80 over
// lib/networks/resnet.py:200-220) as one launch sequence on the caller's stream:
// 25 wgmma convolutions (conv_tc.cu, conv_col.cu; the stem as a 4x4 conv on the space-to-depth image) +
// image packing / max-pool / 3 upsamplings / head (backbone_aux.cu).  Eval mode only: BatchNorm is folded
// into the packed weights by the host layer (pvnet_b200/model_repository.py).  Activations are NHWC fp32
// (TF32-rounded where they feed a tensor-core conv); every torch.cat of the decoder is replaced by
// producers writing into channel slices of one buffer:
//
//   C8 [b,H/8,W/8, fc+128]   xfc -> [0,fc)        x8s (layer2) -> [fc,fc+128)
//   C4 [b,H/4,W/4, s8+64]    up(conv8s) -> [0,s8) x4s (layer1) -> [s8,s8+64)
//   C2 [b,H/2,W/2, s4+64]    up(conv4s) -> [0,s4) x2s (stem)   -> [s4,s4+64)
//   C1 [b,H,  W,   s2]       up(conv2s), followed by [b,H,W,8]: image (3 channels, zeros to 8); convraw.0
//                            reads the two dense parts as its two sources (ConvDesc::in2)
#include "conv_tc.cuh"

#include <vector>

using namespace pvnet;

// conv slots, in execution order.  Slot 0 is the stem as a 4x4 conv on the space-to-depth image; the last (head)
// runs in convraw.0's epilogue or as k_head.
enum {
    CV_STEM = 0,
    CV_L1_0_C1, CV_L1_0_C2, CV_L1_1_C1, CV_L1_1_C2,
    CV_L2_0_C1, CV_L2_0_DS, CV_L2_0_C2, CV_L2_1_C1, CV_L2_1_C2,
    CV_L3_0_C1, CV_L3_0_DS, CV_L3_0_C2, CV_L3_1_C1, CV_L3_1_C2,
    CV_L4_0_C1, CV_L4_0_DS, CV_L4_0_C2, CV_L4_1_C1, CV_L4_1_C2,
    CV_FC, CV_CONV8S, CV_CONV4S, CV_CONV2S, CV_CONVRAW0, CV_HEAD,
    CV_COUNT
};

struct pvnet_backbone {
    int ver_dim, seg_dim, fc, s8, s4, s2, raw;
    const float *w[CV_COUNT];
    const float *bias[CV_COUNT];
    // cached plan for one (b,h,w,workspace,in,out) combination
    int pb = 0, ph = 0, pw = 0;
    const void *p_ws = nullptr;
    std::vector<unsigned char> plans;   // CV_COUNT slots of plan_stride() bytes
    bool use_col[CV_COUNT] = {};         // slot runs on the persistent column kernel (conv_col.cu)
    bool head_fused = false;             // convraw.3 + argmax run inside convraw.0's epilogue
    int out_nhwc = 0;                    // output layout: 0 = [b,C,H,W] (reference), 1 = pixel-major [b,H,W,C]
};

// where the image comes from: float32 NCHW (already normalised) or raw uint8 HWC + mean/std
struct ImageSrc {
    const void *ptr;
    int is_u8;
    float mean[3], std[3];
};

static size_t plan_stride()
{
    const size_t a = conv_plan_size(), b = conv_col_plan_size();
    return ((a > b ? a : b) + 63) / 64 * 64;
}

namespace {

struct Buffers {
    float *S2D, *C1, *R0, *C2, *U2, *P, *A1, *B1, *C4, *U4, *A2, *D2, *B2, *C8, *U8, *A3, *D3, *B3, *E3, *A4, *D4, *B4, *E4;
    size_t bytes;
};

Buffers carve_buffers(const pvnet_backbone *m, void *ws, int b, int h, int w)
{
    Carver c(ws);
    Buffers B;
    const size_t p1 = (size_t)b * h * w, p2 = p1 / 4, p4 = p1 / 16, p8 = p1 / 64;
    B.S2D = c.take<float>(p2 * 16);
    B.C1 = c.take<float>(p1 * (m->s2 + 8));
    B.R0 = c.take<float>(p1 * m->raw);
    B.C2 = c.take<float>(p2 * (m->s4 + 64));
    B.U2 = c.take<float>(p2 * m->s2);
    B.P = c.take<float>(p4 * 64);
    B.A1 = c.take<float>(p4 * 64);
    B.B1 = c.take<float>(p4 * 64);
    B.C4 = c.take<float>(p4 * (m->s8 + 64));
    B.U4 = c.take<float>(p4 * m->s4);
    B.A2 = c.take<float>(p8 * 128);
    B.D2 = c.take<float>(p8 * 128);
    B.B2 = c.take<float>(p8 * 128);
    B.C8 = c.take<float>(p8 * (m->fc + 128));
    B.U8 = c.take<float>(p8 * m->s8);
    B.A3 = c.take<float>(p8 * 256);
    B.D3 = c.take<float>(p8 * 256);
    B.B3 = c.take<float>(p8 * 256);
    B.E3 = c.take<float>(p8 * 256);
    B.A4 = c.take<float>(p8 * 512);
    B.D4 = c.take<float>(p8 * 512);
    B.B4 = c.take<float>(p8 * 512);
    B.E4 = c.take<float>(p8 * 512);
    B.bytes = align_up(c.off, 256);
    return B;
}

ConvDesc cd(const pvnet_backbone *m, int slot, const float *in, int in_cs, int in_co, int cin, float *out, int out_cs,
            int out_co, int cout, int b, int H, int W, int k, int stride, int dil, int act, const float *res = nullptr,
            int res_cs = 0, int res_co = 0, int round_out = 1)
{
    ConvDesc d;
    d.in = in;
    d.in_cs = in_cs;
    d.in_co = in_co;
    d.Cin = cin;
    d.w = m->w[slot];
    d.bias = m->bias[slot];
    d.res = res;
    d.res_cs = res_cs;
    d.res_co = res_co;
    d.out = out;
    d.out_cs = out_cs;
    d.out_co = out_co;
    d.Cout = cout;
    d.b = b;
    d.H = H;
    d.W = W;
    d.ksize = k;
    d.stride = stride;
    d.dilation = dil;
    d.act = act;
    d.round_out = round_out;
    return d;
}

int build_plans(pvnet_backbone *m, const Buffers &B, int b, int h, int w)
{
    const size_t ps = plan_stride();
    m->plans.assign(ps * CV_COUNT, 0);
    m->head_fused = false;
    auto plan = [&](int slot, const ConvDesc &d) {
        void *st = m->plans.data() + ps * slot;
        const bool col = conv_col_eligible(d);
        m->use_col[slot] = col;
        if (!col) return conv_plan_at(d, st);
        if (slot == CV_CONVRAW0 && m->raw == 32 && m->seg_dim + m->ver_dim <= 32) {
            // fuse convraw.3 + argmax into the epilogue; pointers are patched per forward call
            HeadDesc hd{m->w[CV_HEAD], m->bias[CV_HEAD], reinterpret_cast<float *>(0x10), nullptr, 8, m->seg_dim,
                        m->seg_dim + m->ver_dim};
            m->head_fused = true;
            return conv_col_plan_at(d, &hd, st);
        }
        return conv_col_plan_at(d, nullptr, st);
    };
    const int h2 = h / 2, w2 = w / 2, h4 = h / 4, w4 = w / 4, h8 = h / 8, w8 = w / 8;
    const int c4s = m->s8 + 64, c8s = m->fc + 128, c2s = m->s4 + 64;
    int rc = 0;
    // stem (resnet.py:201-203) as a 4x4 stride-1 conv on the 2x2 space-to-depth image
    if ((rc = plan(CV_STEM, cd(m, CV_STEM, B.S2D, 16, 0, 16, B.C2, c2s, m->s4, 64, b, h2, w2, 4, 1, 1, 1)))) return rc;
    // layer1 (resnet.py:206): two BasicBlocks at 1/4 resolution
    if ((rc = plan(CV_L1_0_C1, cd(m, CV_L1_0_C1, B.P, 64, 0, 64, B.A1, 64, 0, 64, b, h4, w4, 3, 1, 1, 1)))) return rc;
    if ((rc = plan(CV_L1_0_C2, cd(m, CV_L1_0_C2, B.A1, 64, 0, 64, B.B1, 64, 0, 64, b, h4, w4, 3, 1, 1, 1, B.P, 64, 0)))) return rc;
    if ((rc = plan(CV_L1_1_C1, cd(m, CV_L1_1_C1, B.B1, 64, 0, 64, B.A1, 64, 0, 64, b, h4, w4, 3, 1, 1, 1)))) return rc;
    if ((rc = plan(CV_L1_1_C2, cd(m, CV_L1_1_C2, B.A1, 64, 0, 64, B.C4, c4s, m->s8, 64, b, h4, w4, 3, 1, 1, 1, B.B1, 64, 0)))) return rc;
    // layer2 (resnet.py:207): stride 2 into 1/8 resolution
    if ((rc = plan(CV_L2_0_C1, cd(m, CV_L2_0_C1, B.C4, c4s, m->s8, 64, B.A2, 128, 0, 128, b, h4, w4, 3, 2, 1, 1)))) return rc;
    if ((rc = plan(CV_L2_0_DS, cd(m, CV_L2_0_DS, B.C4, c4s, m->s8, 64, B.D2, 128, 0, 128, b, h4, w4, 1, 2, 1, 0)))) return rc;
    if ((rc = plan(CV_L2_0_C2, cd(m, CV_L2_0_C2, B.A2, 128, 0, 128, B.B2, 128, 0, 128, b, h8, w8, 3, 1, 1, 1, B.D2, 128, 0)))) return rc;
    if ((rc = plan(CV_L2_1_C1, cd(m, CV_L2_1_C1, B.B2, 128, 0, 128, B.A2, 128, 0, 128, b, h8, w8, 3, 1, 1, 1)))) return rc;
    if ((rc = plan(CV_L2_1_C2, cd(m, CV_L2_1_C2, B.A2, 128, 0, 128, B.C8, c8s, m->fc, 128, b, h8, w8, 3, 1, 1, 1, B.B2, 128, 0)))) return rc;
    // layer3 (resnet.py:208): stride replaced by dilation 2 (resnet.py:173-183)
    if ((rc = plan(CV_L3_0_C1, cd(m, CV_L3_0_C1, B.C8, c8s, m->fc, 128, B.A3, 256, 0, 256, b, h8, w8, 3, 1, 2, 1)))) return rc;
    if ((rc = plan(CV_L3_0_DS, cd(m, CV_L3_0_DS, B.C8, c8s, m->fc, 128, B.D3, 256, 0, 256, b, h8, w8, 1, 1, 1, 0)))) return rc;
    if ((rc = plan(CV_L3_0_C2, cd(m, CV_L3_0_C2, B.A3, 256, 0, 256, B.B3, 256, 0, 256, b, h8, w8, 3, 1, 2, 1, B.D3, 256, 0)))) return rc;
    if ((rc = plan(CV_L3_1_C1, cd(m, CV_L3_1_C1, B.B3, 256, 0, 256, B.A3, 256, 0, 256, b, h8, w8, 3, 1, 2, 1)))) return rc;
    if ((rc = plan(CV_L3_1_C2, cd(m, CV_L3_1_C2, B.A3, 256, 0, 256, B.E3, 256, 0, 256, b, h8, w8, 3, 1, 2, 1, B.B3, 256, 0)))) return rc;
    // layer4 (resnet.py:209): dilation 4
    if ((rc = plan(CV_L4_0_C1, cd(m, CV_L4_0_C1, B.E3, 256, 0, 256, B.A4, 512, 0, 512, b, h8, w8, 3, 1, 4, 1)))) return rc;
    if ((rc = plan(CV_L4_0_DS, cd(m, CV_L4_0_DS, B.E3, 256, 0, 256, B.D4, 512, 0, 512, b, h8, w8, 1, 1, 1, 0)))) return rc;
    if ((rc = plan(CV_L4_0_C2, cd(m, CV_L4_0_C2, B.A4, 512, 0, 512, B.B4, 512, 0, 512, b, h8, w8, 3, 1, 4, 1, B.D4, 512, 0)))) return rc;
    if ((rc = plan(CV_L4_1_C1, cd(m, CV_L4_1_C1, B.B4, 512, 0, 512, B.A4, 512, 0, 512, b, h8, w8, 3, 1, 4, 1)))) return rc;
    if ((rc = plan(CV_L4_1_C2, cd(m, CV_L4_1_C2, B.A4, 512, 0, 512, B.E4, 512, 0, 512, b, h8, w8, 3, 1, 4, 1, B.B4, 512, 0)))) return rc;
    // fc (model_repository.py:22-26): 3x3 conv + BN + ReLU -> xfc
    if ((rc = plan(CV_FC, cd(m, CV_FC, B.E4, 512, 0, 512, B.C8, c8s, 0, m->fc, b, h8, w8, 3, 1, 1, 1)))) return rc;
    // decoder (model_repository.py:66-76): LeakyReLU(0.1)
    if ((rc = plan(CV_CONV8S, cd(m, CV_CONV8S, B.C8, c8s, 0, c8s, B.U8, m->s8, 0, m->s8, b, h8, w8, 3, 1, 1, 2)))) return rc;
    if ((rc = plan(CV_CONV4S, cd(m, CV_CONV4S, B.C4, c4s, 0, c4s, B.U4, m->s4, 0, m->s4, b, h4, w4, 3, 1, 1, 2)))) return rc;
    if ((rc = plan(CV_CONV2S, cd(m, CV_CONV2S, B.C2, c2s, 0, c2s, B.U2, m->s2, 0, m->s2, b, h2, w2, 3, 1, 1, 2)))) return rc;
    // convraw.0 reads cat(upsampled features [s2], image [3 -> 8]) from two dense buffers (the first p1*s2 and the
    // next p1*8 floats of C1) through two tensor maps: a 32-byte image slice inside every 160-byte record made both
    // producers write at ~2 TB/s.
    ConvDesc draw = cd(m, CV_CONVRAW0, B.C1, m->s2, 0, m->s2, B.R0, m->raw, 0, m->raw, b, h, w, 3, 1, 1, 2, nullptr, 0, 0,
                       /*round_out=*/0);
    draw.in2 = B.C1 + (size_t)b * h * w * m->s2;
    draw.in2_cs = 8;
    draw.Cin2 = 8;
    if ((rc = plan(CV_CONVRAW0, draw))) return rc;
    return PVNET_OK;
}

}  // namespace

extern "C" {

int pvnet_backbone_create(int ver_dim, int seg_dim, int fcdim, int s8dim, int s4dim, int s2dim, int raw_dim,
                          pvnet_backbone_t **out)
{
    PV_CHECK_ARG(out, "null out pointer");
    PV_CHECK_ARG(ver_dim >= 0 && seg_dim >= 1 && ver_dim + seg_dim <= 64, "seg_dim+ver_dim must be in [1,64]");
    PV_CHECK_ARG(fcdim % 32 == 0 && s8dim % 32 == 0 && s4dim % 32 == 0 && s2dim % 32 == 0 && fcdim > 0 &&
                     s8dim > 0 && s4dim > 0 && s2dim > 0,
                 "fcdim/s8dim/s4dim/s2dim must be positive multiples of 32");
    PV_CHECK_ARG(raw_dim == 32, "raw_dim must be 32 (head kernel)");
    PV_CHECK_ARG(fcdim <= 512 && s8dim <= 512 && s4dim <= 512 && s2dim <= 512, "decoder widths above 512 unsupported");
    pvnet_backbone *m = new pvnet_backbone();
    m->ver_dim = ver_dim;
    m->seg_dim = seg_dim;
    m->fc = fcdim;
    m->s8 = s8dim;
    m->s4 = s4dim;
    m->s2 = s2dim;
    m->raw = raw_dim;
    for (int i = 0; i < CV_COUNT; ++i) m->w[i] = m->bias[i] = nullptr;
    *out = m;
    return PVNET_OK;
}

void pvnet_backbone_destroy(pvnet_backbone_t *m) { delete m; }

int pvnet_backbone_num_convs(void) { return CV_COUNT; }

int pvnet_backbone_set_output_layout(pvnet_backbone_t *m, int pixel_major)
{
    PV_CHECK_ARG(m, "null handle");
    m->out_nhwc = pixel_major ? 1 : 0;
    return PVNET_OK;
}

int pvnet_backbone_set_conv(pvnet_backbone_t *m, int slot, const float *w_packed, const float *bias)
{
    PV_CHECK_ARG(m, "null handle");
    PV_CHECK_ARG(slot >= 0 && slot < CV_COUNT, "conv slot %d out of range", slot);
    PV_CHECK_ARG(w_packed && bias, "null weight/bias pointer");
    m->w[slot] = w_packed;
    m->bias[slot] = bias;
    m->p_ws = nullptr;   // cached tensor maps point at the old weights
    return PVNET_OK;
}

int pvnet_backbone_workspace_bytes(const pvnet_backbone_t *m, int b, int h, int w, size_t *bytes)
{
    PV_CHECK_ARG(m && bytes, "null pointer");
    PV_CHECK_ARG(b >= 1 && h >= 16 && w >= 16 && h % 8 == 0 && w % 8 == 0, "image size must be a multiple of 8");
    *bytes = carve_buffers(m, nullptr, b, h, w).bytes + 256;
    return PVNET_OK;
}

// The forward pass as an ordered list of stages (one kernel launch each).
namespace {
enum StageKind { ST_PACK, ST_POOL, ST_CONV, ST_UP8, ST_UP4, ST_UP2, ST_HEAD };
struct Stage {
    StageKind kind;
    int slot;
    const char *name;
};
const Stage kStages[] = {
    {ST_PACK, -1, "image: space-to-depth + NHWC slice packing"},
    {ST_CONV, CV_STEM, "stem conv1+bn1+relu"},
    {ST_POOL, -1, "maxpool 3x3/2"},
    {ST_CONV, CV_L1_0_C1, "layer1.0.conv1"}, {ST_CONV, CV_L1_0_C2, "layer1.0.conv2"},
    {ST_CONV, CV_L1_1_C1, "layer1.1.conv1"}, {ST_CONV, CV_L1_1_C2, "layer1.1.conv2"},
    {ST_CONV, CV_L2_0_C1, "layer2.0.conv1 (s2)"}, {ST_CONV, CV_L2_0_DS, "layer2.0.downsample (1x1 s2)"},
    {ST_CONV, CV_L2_0_C2, "layer2.0.conv2"}, {ST_CONV, CV_L2_1_C1, "layer2.1.conv1"},
    {ST_CONV, CV_L2_1_C2, "layer2.1.conv2"},
    {ST_CONV, CV_L3_0_C1, "layer3.0.conv1 (d2)"}, {ST_CONV, CV_L3_0_DS, "layer3.0.downsample (1x1)"},
    {ST_CONV, CV_L3_0_C2, "layer3.0.conv2 (d2)"}, {ST_CONV, CV_L3_1_C1, "layer3.1.conv1 (d2)"},
    {ST_CONV, CV_L3_1_C2, "layer3.1.conv2 (d2)"},
    {ST_CONV, CV_L4_0_C1, "layer4.0.conv1 (d4)"}, {ST_CONV, CV_L4_0_DS, "layer4.0.downsample (1x1)"},
    {ST_CONV, CV_L4_0_C2, "layer4.0.conv2 (d4)"}, {ST_CONV, CV_L4_1_C1, "layer4.1.conv1 (d4)"},
    {ST_CONV, CV_L4_1_C2, "layer4.1.conv2 (d4)"},
    {ST_CONV, CV_FC, "fc.0"}, {ST_CONV, CV_CONV8S, "conv8s.0"},
    {ST_UP8, -1, "upsample 1/8->1/4"}, {ST_CONV, CV_CONV4S, "conv4s.0"},
    {ST_UP4, -1, "upsample 1/4->1/2"}, {ST_CONV, CV_CONV2S, "conv2s.0"},
    {ST_UP2, -1, "upsample 1/2->1"}, {ST_CONV, CV_CONVRAW0, "convraw.0"},
    {ST_HEAD, CV_HEAD, "convraw.3 1x1 + argmax head (fp32)"},
};
constexpr int kNumStages = (int)(sizeof(kStages) / sizeof(kStages[0]));

int prepare(pvnet_backbone *m, const ImageSrc &img, int b, int h, int w, float *out_nchw, void *mask_out,
            int mask_elem_size, void *workspace, size_t workspace_bytes, Buffers *B)
{
    PV_CHECK_ARG(m && img.ptr && out_nchw && workspace, "null pointer");
    PV_CHECK_ARG(b >= 1 && h >= 16 && w >= 16 && h % 8 == 0 && w % 8 == 0, "image size must be a multiple of 8");
    PV_CHECK_ARG(!mask_out || mask_elem_size == 1 || mask_elem_size == 8, "mask element size must be 1 or 8");
    for (int i = 0; i < CV_COUNT; ++i)
        if (!m->w[i] || !m->bias[i]) {
            set_error("conv slot %d has no weights (pvnet_backbone_set_conv)", i);
            return PVNET_E_STATE;
        }
    PV_CHECK_ARG((uintptr_t)workspace % 256 == 0, "workspace must be 256-byte aligned");
    *B = carve_buffers(m, workspace, b, h, w);
    if (workspace_bytes < B->bytes) {
        set_error("workspace %zu < %zu bytes", workspace_bytes, B->bytes);
        return PVNET_E_WORKSPACE;
    }
    if (m->p_ws != workspace || m->pb != b || m->ph != h || m->pw != w) {
        int rc = build_plans(m, *B, b, h, w);
        if (rc) return rc;
        m->p_ws = workspace;
        m->pb = b;
        m->ph = h;
        m->pw = w;
    }
    return PVNET_OK;
}

int run_stage(pvnet_backbone *m, const Stage &st, const Buffers &B, const ImageSrc &img, int b, int h, int w,
              float *out_nchw, void *mask_out, int mask_elem_size, cudaStream_t s)
{
    const int h2 = h / 2, w2 = w / 2, h4 = h / 4, w4 = w / 4, h8 = h / 8, w8 = w / 8;
    const int c4s = m->s8 + 64, c2s = m->s4 + 64;
    switch (st.kind) {
    case ST_PACK:
        return launch_s2d_pack(img.ptr, img.is_u8, img.mean, img.std, B.S2D, B.C1 + (size_t)b * h * w * m->s2, b, h, w, 8, 0,
                               s);
    case ST_POOL: return launch_maxpool(B.C2, B.P, b, h2, w2, 64, c2s, m->s4, s);
    case ST_CONV: {
        unsigned char *pl = m->plans.data() + plan_stride() * st.slot;
        if (!m->use_col[st.slot]) return conv_launch_at(pl, s);
        if (st.slot == CV_CONVRAW0 && m->head_fused) conv_col_set_head_ptrs(pl, out_nchw, mask_out, mask_elem_size, m->out_nhwc);
        return conv_col_launch_at(pl, s);
    }
    case ST_UP8: return launch_upsample2x(B.U8, B.C4, b, h8, w8, m->s8, c4s, 0, s);
    case ST_UP4: return launch_upsample2x(B.U4, B.C2, b, h4, w4, m->s4, c2s, 0, s);
    case ST_UP2: return launch_upsample2x(B.U2, B.C1, b, h2, w2, m->s2, m->s2, 0, s);
    case ST_HEAD:
        if (m->head_fused) return PVNET_OK;    // already written by convraw.0's epilogue
        return launch_head(B.R0, m->w[CV_HEAD], m->bias[CV_HEAD], out_nchw, mask_out, mask_elem_size, m->seg_dim,
                           m->seg_dim + m->ver_dim, b, h, w, m->out_nhwc, s);
    }
    return PVNET_E_INVALID;
}
}  // namespace

int pvnet_backbone_num_stages(void) { return kNumStages; }

const char *pvnet_backbone_stage_name(int stage)
{
    return (stage >= 0 && stage < kNumStages) ? kStages[stage].name : "";
}

int pvnet_backbone_run_stage(pvnet_backbone_t *m, int stage, const float *image_nchw, int b, int h, int w,
                             float *out_nchw, void *mask_out, int mask_elem_size, void *workspace,
                             size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(stage >= 0 && stage < kNumStages, "stage %d out of range", stage);
    Buffers B;
    const ImageSrc img{image_nchw, 0, {0, 0, 0}, {1, 1, 1}};
    int rc = prepare(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, &B);
    if (rc) return rc;
    return run_stage(m, kStages[stage], B, img, b, h, w, out_nchw, mask_out, mask_elem_size, (cudaStream_t)stream);
}

static int forward_impl(pvnet_backbone_t *m, const ImageSrc &img, int b, int h, int w, float *out_nchw, void *mask_out,
                        int mask_elem_size, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    Buffers B;
    int rc = prepare(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, &B);
    if (rc) return rc;
    for (int i = 0; i < kNumStages; ++i)
        if ((rc = run_stage(m, kStages[i], B, img, b, h, w, out_nchw, mask_out, mask_elem_size, (cudaStream_t)stream)))
            return rc;
    return PVNET_OK;
}

int pvnet_backbone_forward_u8(pvnet_backbone_t *m, const uint8_t *image_hwc, const float mean[3], const float std[3],
                              int b, int h, int w, float *out_nchw, void *mask_out, int mask_elem_size,
                              void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(mean && std, "null mean/std");
    PV_CHECK_ARG(std[0] != 0.f && std[1] != 0.f && std[2] != 0.f, "zero std");
    PV_CHECK_ARG((reinterpret_cast<uintptr_t>(image_hwc) & 1) == 0 && w % 2 == 0, "uint8 image must be 2-byte aligned");
    const ImageSrc img{image_hwc, 1, {mean[0], mean[1], mean[2]}, {std[0], std[1], std[2]}};
    return forward_impl(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, stream);
}

int pvnet_backbone_forward(pvnet_backbone_t *m, const float *image_nchw, int b, int h, int w, float *out_nchw,
                           void *mask_out, int mask_elem_size, void *workspace, size_t workspace_bytes,
                           pvnet_stream_t stream)
{
    const ImageSrc img{image_nchw, 0, {0, 0, 0}, {1, 1, 1}};
    return forward_impl(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, stream);
}

}  // extern "C"
