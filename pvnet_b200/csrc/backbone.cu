// backbone.cu -- the eval forward of Resnet18_8s / Resnet34_8s / Resnet50_8s (lib/networks/model_repository.py over
// lib/networks/resnet.py:116-220) as one launch sequence on the caller's stream: the wgmma convolutions (conv_tc.cu,
// conv_col.cu; the stem as a 4x4 conv on the space-to-depth image) + image packing / max-pool / 3 upsamplings / head
// (backbone_aux.cu).  Eval mode only: BatchNorm is folded into the packed weights by the host layer
// (pvnet_b200/model_repository.py).  Activations are NHWC fp32 (TF32-rounded where they feed a tensor-core conv);
// every torch.cat of the decoder is replaced by producers writing into channel slices of one buffer
// (x4c / x8c: the channels of layer1 / layer2's output, 64 / 128 for BasicBlock trunks, 256 / 512 for Bottleneck):
//
//   C8 [b,H/8,W/8, fc+x8c]   xfc -> [0,fc)        x8s (layer2) -> [fc,fc+x8c)
//   C4 [b,H/4,W/4, s8+x4c]   up(conv8s) -> [0,s8) x4s (layer1) -> [s8,s8+x4c)
//   C2 [b,H/2,W/2, s4+64]    up(conv4s) -> [0,s4) x2s (stem)   -> [s4,s4+64)
//   C1 [b,H,  W,   s2]       up(conv2s), followed by [b,H,W,8]: image (3 channels, zeros to 8); convraw.0
//                            reads the two dense parts as its two sources (ConvDesc::in2)
//
// The plan -- conv slots, workspace buffers, stage list -- is generated once per handle from the trunk description
// (block kind, blocks per stage, decoder widths) and the decoder kind by `generate`; for the 2-2-2-2 BasicBlock trunk
// and the full-resolution decoder it is the Resnet18_8s plan: slots, buffer order and sizes, and launches.
// The half-resolution decoder (Resnet50_8s_2o, model_repository.py:158-224) ends at conv2s: C1, R0 and the x2
// upsampling are gone, and conv2s.0 reads C2 plus X [b,H/2,W/2,8] (x_ds, 3 channels, zeros to 8; written by the
// image pack) as its second source, into U2, which the 1x1 head reads at H/2 x W/2.
// The detector kind (Resnet18_8s_detector / _v2, model_repository.py:302-331) has no decoder: the trunk up to layer4
// (v1) or layer2 (v2), every stage writing plain buffers (no concatenation slices), then the 3x3 one-channel score
// head (head3x3.cu) on the last stage's output at H/8 x W/8.
#include "conv_tc.cuh"

#include <string>
#include <vector>

using namespace pvnet;

namespace {

enum StageKind { ST_PACK, ST_POOL, ST_CONV, ST_UP8, ST_UP4, ST_UP2, ST_HEAD, ST_SCORE };

struct Stage {
    StageKind kind;
    int slot;
    std::string name;
};

// one workspace buffer: NHWC fp32 at resolution 1/2^level, `ch` channels per pixel
struct BufSpec {
    int level, ch;
};

// one convolution of the plan; buffers are indices into pvnet_backbone::bufs
struct Layer {
    int in, in_cs, in_co, cin;
    int out, out_cs, out_co, cout;
    int res = -1, res_cs = 0, res_co = 0;
    int level;                  // input resolution 1/2^level
    int k, stride, dil, act;
    int round_out = 1;
    bool image_src = false;     // convraw.0: second source = the 8-channel image slice behind C1's first part
    int in2 = -1;               // conv2s.0 of the half-resolution decoder: second source = this dense 8-channel buffer
};

}  // namespace

struct pvnet_backbone {
    int ver_dim, seg_dim, fc, s8, s4, s2, raw;   // raw: the head's input width (s2 in the half-resolution decoder)
    int half = 0;                        // decoder kind: 1 = Resnet50_8s_2o's, output at H/2 x W/2
    int last_stage = 0;                  // decoder kind: 4 / 2 = the detectors' score head on layer4 / layer2's output
    int nconv = 0;                       // conv slots, the head included (the last slot)
    std::vector<const float *> w, bias;
    std::vector<BufSpec> bufs;           // in carving order
    std::vector<Layer> layers;           // by slot, the head excluded
    std::vector<Stage> stages;
    int bS2D, bC1 = -1, bR0 = -1, bX = -1, bC2, bU2 = -1, bP, bC4 = -1, bU4 = -1, bC8 = -1, bU8 = -1;   // buffers the
    int bFeat = -1, feat_c = 0;          // non-conv stages use; the score head's input and its channels (detectors)
    int c2s, c4s, c8s;                   // channel strides of the concatenation buffers
    // cached plan for one (b,h,w,workspace,in,out) combination
    int pb = 0, ph = 0, pw = 0;
    const void *p_ws = nullptr;
    std::vector<unsigned char> plans;    // nconv slots of plan_stride() bytes
    std::vector<unsigned char> use_col;  // slot runs on the persistent column kernel (conv_col.cu)
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

// The plan of resnet.py's ResNet(block, blocks, output_stride=8) under model_repository.py's decoder.  Stage rule
// (resnet.py:167-198): a stage that would take the output stride past 8 keeps stride 1 and multiplies the dilation
// instead, for every block of it; the 1x1 downsample is never dilated.  BasicBlock: conv1 (3x3, the stride) ->
// conv2 (3x3) + skip + ReLU.  Bottleneck (expansion 4): conv1 (1x1) -> conv2 (3x3, the stride) -> conv3 (1x1) + skip
// + ReLU.  The downsample runs just before the conv whose epilogue adds it.  Within a stage the block outputs
// alternate between two buffers so that the last block writes the stage's output: layer1 / layer2 straight into
// their concatenation slices, layer3 / layer4 into E.  The detector kind stops after stage `last_stage`, and every
// stage writes its own E.
void generate(pvnet_backbone *m, int bottleneck, const int blocks[4])
{
    const bool det = m->last_stage > 0;
    auto buf = [&](int level, int ch) {
        m->bufs.push_back({level, ch});
        return (int)m->bufs.size() - 1;
    };
    auto conv = [&](const Layer &l, const std::string &name) {
        m->stages.push_back({ST_CONV, (int)m->layers.size(), name});
        m->layers.push_back(l);
    };
    const int e = bottleneck ? 4 : 1;
    m->c2s = det ? 64 : m->s4 + 64;
    m->c4s = m->s8 + 64 * e;
    m->c8s = m->fc + 128 * e;
    m->bS2D = buf(1, 16);
    if (m->half) {
        m->bX = buf(1, 8);
    } else if (!det) {
        m->bC1 = buf(0, m->s2 + 8);
        m->bR0 = buf(0, m->raw);
    }
    m->bC2 = buf(1, m->c2s);
    if (!det) m->bU2 = buf(1, m->s2);
    m->bP = buf(2, 64);
    m->stages.push_back({ST_PACK, -1, det ? "image: space-to-depth packing"
                                          : "image: space-to-depth + NHWC slice packing"});
    // stem (resnet.py:201-203) as a 4x4 stride-1 conv on the 2x2 space-to-depth image
    conv({m->bS2D, 16, 0, 16, m->bC2, m->c2s, m->s4, 64, -1, 0, 0, 1, 4, 1, 1, 1}, "stem conv1+bn1+relu");
    m->stages.push_back({ST_POOL, -1, "maxpool 3x3/2"});
    int x = m->bP, x_cs = 64, x_co = 0, x_c = 64, level = 2;
    int cur_stride = 4, dil = 1;
    for (int s = 0; s < (det ? m->last_stage : 4); ++s) {
        const int planes = 64 << s, outc = planes * e, n = blocks[s];
        int stride = s == 0 ? 1 : 2;
        const bool has_ds = stride != 1 || x_c != outc;
        if (has_ds) {
            if (cur_stride == 8) {
                dil *= stride;
                stride = 1;
            } else {
                cur_stride *= stride;
            }
        }
        const int olevel = level + (stride == 2 ? 1 : 0);
        const int A = buf(bottleneck ? level : olevel, planes);
        const int M = bottleneck ? buf(olevel, planes) : -1;
        const int D = has_ds ? buf(olevel, outc) : -1;
        const int B = buf(olevel, outc);
        const int E = (det || s >= 2 || n > 2) ? buf(olevel, outc) : -1;
        int out, out_cs, out_co;
        if (det) {
            out = E;
            out_cs = outc;
            out_co = 0;
        } else if (s == 0) {
            m->bC4 = out = buf(2, m->c4s);
            m->bU4 = buf(2, m->s4);
            out_cs = m->c4s;
            out_co = m->s8;
        } else if (s == 1) {
            m->bC8 = out = buf(3, m->c8s);
            m->bU8 = buf(3, m->s8);
            out_cs = m->c8s;
            out_co = m->fc;
        } else {
            out = E;
            out_cs = outc;
            out_co = 0;
        }
        const std::string dtag = dil > 1 ? " (d" + std::to_string(dil) + ")" : "";
        for (int i = 0; i < n; ++i) {
            const std::string pre = "layer" + std::to_string(s + 1) + "." + std::to_string(i) + ".";
            const int st = i == 0 ? stride : 1, left = n - 1 - i;
            const int y = left == 0 ? out : (left % 2 ? B : E);
            const int y_cs = left == 0 ? out_cs : outc, y_co = left == 0 ? out_co : 0;
            const std::string tag3 = st == 2 ? " (s2)" : dtag;
            int r = x, r_cs = x_cs, r_co = x_co;
            auto downsample = [&]() {
                conv({x, x_cs, x_co, x_c, D, outc, 0, outc, -1, 0, 0, level, 1, st, 1, 0},
                     pre + (st == 2 ? "downsample (1x1 s2)" : "downsample (1x1)"));
                r = D, r_cs = outc, r_co = 0;
            };
            if (!bottleneck) {
                conv({x, x_cs, x_co, x_c, A, planes, 0, planes, -1, 0, 0, level, 3, st, dil, 1}, pre + "conv1" + tag3);
                if (i == 0 && has_ds) downsample();
                conv({A, planes, 0, planes, y, y_cs, y_co, outc, r, r_cs, r_co, olevel, 3, 1, dil, 1},
                     pre + "conv2" + dtag);
            } else {
                conv({x, x_cs, x_co, x_c, A, planes, 0, planes, -1, 0, 0, level, 1, 1, 1, 1}, pre + "conv1 (1x1)");
                conv({A, planes, 0, planes, M, planes, 0, planes, -1, 0, 0, level, 3, st, dil, 1}, pre + "conv2" + tag3);
                if (i == 0 && has_ds) downsample();
                conv({M, planes, 0, planes, y, y_cs, y_co, outc, r, r_cs, r_co, olevel, 1, 1, 1, 1}, pre + "conv3 (1x1)");
            }
            x = y, x_cs = y_cs, x_co = y_co, x_c = outc, level = olevel;
        }
    }
    if (det) {
        m->bFeat = x;
        m->feat_c = x_c;
        m->nconv = (int)m->layers.size() + 1;
        m->stages.push_back({ST_SCORE, m->nconv - 1, m->last_stage == 4 ? "fc 3x3 -> 1 score head (fp32)"
                                                                        : "out_conv 3x3 -> 1 score head (fp32)"});
        m->w.assign(m->nconv, nullptr);
        m->bias.assign(m->nconv, nullptr);
        return;
    }
    // fc (model_repository.py: resnet.fc = 3x3 conv + BN + ReLU) -> xfc; decoder with LeakyReLU(0.1)
    conv({x, x_cs, x_co, x_c, m->bC8, m->c8s, 0, m->fc, -1, 0, 0, 3, 3, 1, 1, 1}, "fc.0");
    conv({m->bC8, m->c8s, 0, m->c8s, m->bU8, m->s8, 0, m->s8, -1, 0, 0, 3, 3, 1, 1, 2}, "conv8s.0");
    m->stages.push_back({ST_UP8, -1, "upsample 1/8->1/4"});
    conv({m->bC4, m->c4s, 0, m->c4s, m->bU4, m->s4, 0, m->s4, -1, 0, 0, 2, 3, 1, 1, 2}, "conv4s.0");
    m->stages.push_back({ST_UP4, -1, "upsample 1/4->1/2"});
    if (m->half) {
        // conv2s.0 reads cat[up(conv4s), x2s, x_ds] as C2 and X; its output feeds the fp32 head unrounded
        Layer c2{m->bC2, m->c2s, 0, m->c2s, m->bU2, m->s2, 0, m->s2, -1, 0, 0, 1, 3, 1, 1, 2};
        c2.round_out = 0;
        c2.in2 = m->bX;
        conv(c2, "conv2s.0");
        m->nconv = (int)m->layers.size() + 1;
        m->stages.push_back({ST_HEAD, m->nconv - 1, "conv2s.3 1x1 + argmax head (fp32)"});
        m->w.assign(m->nconv, nullptr);
        m->bias.assign(m->nconv, nullptr);
        return;
    }
    conv({m->bC2, m->c2s, 0, m->c2s, m->bU2, m->s2, 0, m->s2, -1, 0, 0, 1, 3, 1, 1, 2}, "conv2s.0");
    m->stages.push_back({ST_UP2, -1, "upsample 1/2->1"});
    // convraw.0 reads cat(upsampled features [s2], image [3 -> 8]) from two dense buffers (the first p1*s2 and the
    // next p1*8 floats of C1) through two tensor maps: a 32-byte image slice inside every 160-byte record made both
    // producers write at ~2 TB/s.
    Layer raw{m->bC1, m->s2, 0, m->s2, m->bR0, m->raw, 0, m->raw, -1, 0, 0, 0, 3, 1, 1, 2};
    raw.round_out = 0;
    raw.image_src = true;
    conv(raw, "convraw.0");
    m->nconv = (int)m->layers.size() + 1;
    m->stages.push_back({ST_HEAD, m->nconv - 1, "convraw.3 1x1 + argmax head (fp32)"});
    m->w.assign(m->nconv, nullptr);
    m->bias.assign(m->nconv, nullptr);
}

// the Resnet18_8s plan: what the handle-less queries (pvnet_backbone_num_convs, _num_stages, _stage_name) describe
const pvnet_backbone &resnet18_plan()
{
    static const pvnet_backbone r18 = [] {
        pvnet_backbone m;
        m.ver_dim = 18, m.seg_dim = 2, m.fc = 256, m.s8 = 128, m.s4 = 64, m.s2 = 32, m.raw = 32;
        const int blocks[4] = {2, 2, 2, 2};
        generate(&m, 0, blocks);
        return m;
    }();
    return r18;
}

size_t carve_buffers(const pvnet_backbone *m, void *ws, int b, int h, int w, std::vector<float *> *ptrs)
{
    Carver c(ws);
    const size_t p1 = (size_t)b * h * w;
    if (ptrs) ptrs->clear();
    for (const BufSpec &s : m->bufs) {
        float *p = c.take<float>((p1 >> (2 * s.level)) * s.ch);
        if (ptrs) ptrs->push_back(p);
    }
    return align_up(c.off, 256);
}

int build_plans(pvnet_backbone *m, const std::vector<float *> &B, int b, int h, int w)
{
    const size_t ps = plan_stride();
    m->plans.assign(ps * m->nconv, 0);
    m->use_col.assign(m->nconv, 0);
    m->head_fused = false;
    const int head = m->nconv - 1;
    for (int slot = 0; slot < (int)m->layers.size(); ++slot) {
        const Layer &l = m->layers[slot];
        ConvDesc d;
        d.in = B[l.in];
        d.in_cs = l.in_cs;
        d.in_co = l.in_co;
        d.Cin = l.cin;
        d.w = m->w[slot];
        d.bias = m->bias[slot];
        d.res = l.res >= 0 ? B[l.res] : nullptr;
        d.res_cs = l.res_cs;
        d.res_co = l.res_co;
        d.out = B[l.out];
        d.out_cs = l.out_cs;
        d.out_co = l.out_co;
        d.Cout = l.cout;
        d.b = b;
        d.H = h >> l.level;
        d.W = w >> l.level;
        d.ksize = l.k;
        d.stride = l.stride;
        d.dilation = l.dil;
        d.act = l.act;
        d.round_out = l.round_out;
        if (l.image_src) {
            d.in2 = B[l.in] + (size_t)b * h * w * m->s2;
            d.in2_cs = 8;
            d.Cin2 = 8;
        }
        if (l.in2 >= 0) {
            d.in2 = B[l.in2];
            d.in2_cs = 8;
            d.Cin2 = 8;
        }
        void *st = m->plans.data() + ps * slot;
        const bool col = conv_col_eligible(d);
        m->use_col[slot] = col;
        int rc;
        if (!col) {
            rc = conv_plan_at(d, st);
        } else if (l.in2 >= 0 && l.cin % 32 == 0 && l.cout == 64) {
            // conv2s.0 of the half-resolution decoder: 32-channel chunks over C2, X as one 8-channel chunk (s2dim 32
            // keeps the 8-channel-chunk form)
            rc = conv_col_plan_split_at(d, st);
        } else if (l.image_src && m->raw == 32 && m->seg_dim + m->ver_dim <= 32) {
            // fuse convraw.3 + argmax into the epilogue; pointers are patched per forward call
            HeadDesc hd{m->w[head], m->bias[head], reinterpret_cast<float *>(0x10), nullptr, 8, m->seg_dim,
                        m->seg_dim + m->ver_dim};
            m->head_fused = true;
            rc = conv_col_plan_at(d, &hd, st);
        } else {
            rc = conv_col_plan_at(d, nullptr, st);
        }
        if (rc) return rc;
    }
    return PVNET_OK;
}

int check_dims(int ver_dim, int seg_dim, int fcdim, int s8dim, int s4dim, int s2dim, pvnet_backbone_t **out)
{
    PV_CHECK_ARG(out, "null out pointer");
    PV_CHECK_ARG(ver_dim >= 0 && seg_dim >= 1 && ver_dim + seg_dim <= 64, "seg_dim+ver_dim must be in [1,64]");
    PV_CHECK_ARG(fcdim % 32 == 0 && s8dim % 32 == 0 && s4dim % 32 == 0 && s2dim % 32 == 0 && fcdim > 0 &&
                     s8dim > 0 && s4dim > 0 && s2dim > 0,
                 "fcdim/s8dim/s4dim/s2dim must be positive multiples of 32");
    PV_CHECK_ARG(fcdim <= 512 && s8dim <= 512 && s4dim <= 512 && s2dim <= 512, "decoder widths above 512 unsupported");
    return PVNET_OK;
}

pvnet_backbone *make(int bottleneck, const int blocks[4], int ver_dim, int seg_dim, int fcdim, int s8dim, int s4dim,
                     int s2dim, int raw_dim, int half = 0, int last_stage = 0)
{
    pvnet_backbone *m = new pvnet_backbone();
    m->half = half;
    m->last_stage = last_stage;
    m->ver_dim = ver_dim;
    m->seg_dim = seg_dim;
    m->fc = fcdim;
    m->s8 = s8dim;
    m->s4 = s4dim;
    m->s2 = s2dim;
    m->raw = raw_dim;
    generate(m, bottleneck, blocks);
    return m;
}

}  // namespace

extern "C" {

int pvnet_backbone_create(int ver_dim, int seg_dim, int fcdim, int s8dim, int s4dim, int s2dim, int raw_dim,
                          pvnet_backbone_t **out)
{
    if (int rc = check_dims(ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, out)) return rc;
    PV_CHECK_ARG(raw_dim == 32, "raw_dim must be 32 (head kernel)");
    const int blocks[4] = {2, 2, 2, 2};
    *out = make(0, blocks, ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim);
    return PVNET_OK;
}

static int check_trunk(int block_kind, const int *blocks)
{
    PV_CHECK_ARG(block_kind == PVNET_BLOCK_BASIC || block_kind == PVNET_BLOCK_BOTTLENECK,
                 "block kind must be %d (BasicBlock) or %d (Bottleneck), got %d", PVNET_BLOCK_BASIC,
                 PVNET_BLOCK_BOTTLENECK, block_kind);
    PV_CHECK_ARG(blocks, "null block counts");
    for (int s = 0; s < 4; ++s)
        PV_CHECK_ARG(blocks[s] >= 1 && blocks[s] <= 64, "stage %d: %d blocks, must be in [1,64]", s + 1, blocks[s]);
    return PVNET_OK;
}

int pvnet_backbone_create_trunk(int block_kind, const int *blocks, int ver_dim, int seg_dim, int fcdim, int s8dim,
                                int s4dim, int s2dim, int raw_dim, pvnet_backbone_t **out)
{
    if (int rc = check_dims(ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, out)) return rc;
    if (int rc = check_trunk(block_kind, blocks)) return rc;
    PV_CHECK_ARG(raw_dim == 32 || raw_dim == 64, "raw_dim must be 32 or 64 (head kernel), got %d", raw_dim);
    *out = make(block_kind == PVNET_BLOCK_BOTTLENECK, blocks, ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim);
    return PVNET_OK;
}

int pvnet_backbone_create_trunk_2o(int block_kind, const int *blocks, int ver_dim, int seg_dim, int fcdim, int s8dim,
                                   int s4dim, int s2dim, pvnet_backbone_t **out)
{
    if (int rc = check_dims(ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, out)) return rc;
    if (int rc = check_trunk(block_kind, blocks)) return rc;
    PV_CHECK_ARG(s2dim == 32 || s2dim == 64, "s2dim must be 32 or 64 (the head reads conv2s.0's output), got %d",
                 s2dim);
    *out = make(block_kind == PVNET_BLOCK_BOTTLENECK, blocks, ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, s2dim, 1);
    return PVNET_OK;
}

int pvnet_backbone_create_detector(int block_kind, const int *blocks, int last_stage, pvnet_backbone_t **out)
{
    PV_CHECK_ARG(out, "null out pointer");
    if (int rc = check_trunk(block_kind, blocks)) return rc;
    PV_CHECK_ARG(last_stage == 2 || last_stage == 4, "last_stage must be 2 (v2: layer2) or 4 (layer4), got %d",
                 last_stage);
    const int width = (128 << (last_stage - 2)) * (block_kind == PVNET_BLOCK_BOTTLENECK ? 4 : 1);
    PV_CHECK_ARG(width <= 512, "the score head reads at most 512 channels, stage %d has %d", last_stage, width);
    *out = make(block_kind == PVNET_BLOCK_BOTTLENECK, blocks, 0, 1, 0, 0, 0, 0, 0, 0, last_stage);
    return PVNET_OK;
}

int pvnet_backbone_output_scale(const pvnet_backbone_t *m)
{
    return m ? (m->last_stage ? 8 : m->half ? 2 : 1) : -1;
}

void pvnet_backbone_destroy(pvnet_backbone_t *m) { delete m; }

int pvnet_backbone_num_convs(void) { return resnet18_plan().nconv; }

int pvnet_backbone_handle_num_convs(const pvnet_backbone_t *m) { return m ? m->nconv : -1; }

int pvnet_backbone_set_output_layout(pvnet_backbone_t *m, int pixel_major)
{
    PV_CHECK_ARG(m, "null handle");
    m->out_nhwc = pixel_major ? 1 : 0;
    return PVNET_OK;
}

int pvnet_backbone_set_conv(pvnet_backbone_t *m, int slot, const float *w_packed, const float *bias)
{
    PV_CHECK_ARG(m, "null handle");
    PV_CHECK_ARG(slot >= 0 && slot < m->nconv, "conv slot %d out of range", slot);
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
    *bytes = carve_buffers(m, nullptr, b, h, w, nullptr) + 256;
    return PVNET_OK;
}

}  // extern "C"

// The forward pass as an ordered list of stages (one kernel launch each).
namespace {

int prepare(pvnet_backbone *m, const ImageSrc &img, int b, int h, int w, float *out_nchw, void *mask_out,
            int mask_elem_size, void *workspace, size_t workspace_bytes, std::vector<float *> *B)
{
    PV_CHECK_ARG(m && img.ptr && out_nchw && workspace, "null pointer");
    PV_CHECK_ARG(b >= 1 && h >= 16 && w >= 16 && h % 8 == 0 && w % 8 == 0, "image size must be a multiple of 8");
    PV_CHECK_ARG(!mask_out || mask_elem_size == 1 || mask_elem_size == 8, "mask element size must be 1 or 8");
    PV_CHECK_ARG(!mask_out || !m->last_stage, "a detector has no segmentation output: mask must be NULL");
    for (int i = 0; i < m->nconv; ++i)
        if (!m->w[i] || !m->bias[i]) {
            set_error("conv slot %d has no weights (pvnet_backbone_set_conv)", i);
            return PVNET_E_STATE;
        }
    PV_CHECK_ARG((uintptr_t)workspace % 256 == 0, "workspace must be 256-byte aligned");
    const size_t need = carve_buffers(m, workspace, b, h, w, B);
    if (workspace_bytes < need) {
        set_error("workspace %zu < %zu bytes", workspace_bytes, need);
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

int run_stage(pvnet_backbone *m, const Stage &st, const std::vector<float *> &B, const ImageSrc &img, int b, int h,
              int w, float *out_nchw, void *mask_out, int mask_elem_size, cudaStream_t s)
{
    const int h2 = h / 2, w2 = w / 2, h4 = h / 4, w4 = w / 4, h8 = h / 8, w8 = w / 8;
    float *C1 = m->bC1 >= 0 ? B[m->bC1] : nullptr;
    switch (st.kind) {
    case ST_PACK:
        if (m->last_stage)
            return launch_s2d_pack(img.ptr, img.is_u8, img.mean, img.std, B[m->bS2D], nullptr, b, h, w, 8, 0, 0, s);
        if (m->half) return launch_s2d_pack(img.ptr, img.is_u8, img.mean, img.std, B[m->bS2D], B[m->bX], b, h, w, 8, 0, 1, s);
        return launch_s2d_pack(img.ptr, img.is_u8, img.mean, img.std, B[m->bS2D], C1 + (size_t)b * h * w * m->s2, b, h,
                               w, 8, 0, 0, s);
    case ST_POOL: return launch_maxpool(B[m->bC2], B[m->bP], b, h2, w2, 64, m->c2s, m->s4, s);
    case ST_CONV: {
        unsigned char *pl = m->plans.data() + plan_stride() * st.slot;
        if (!m->use_col[st.slot]) return conv_launch_at(pl, s);
        if (m->layers[st.slot].image_src && m->head_fused)
            conv_col_set_head_ptrs(pl, out_nchw, mask_out, mask_elem_size, m->out_nhwc);
        return conv_col_launch_at(pl, s);
    }
    case ST_UP8: return launch_upsample2x(B[m->bU8], B[m->bC4], b, h8, w8, m->s8, m->c4s, 0, s);
    case ST_UP4: return launch_upsample2x(B[m->bU4], B[m->bC2], b, h4, w4, m->s4, m->c2s, 0, s);
    case ST_UP2: return launch_upsample2x(B[m->bU2], C1, b, h2, w2, m->s2, m->s2, 0, s);
    case ST_HEAD:
        if (m->head_fused) return PVNET_OK;    // already written by convraw.0's epilogue
        if (m->half)
            return launch_head(B[m->bU2], m->raw, m->w[st.slot], m->bias[st.slot], out_nchw, mask_out, mask_elem_size,
                               m->seg_dim, m->seg_dim + m->ver_dim, b, h2, w2, m->out_nhwc, s);
        return launch_head(B[m->bR0], m->raw, m->w[st.slot], m->bias[st.slot], out_nchw, mask_out, mask_elem_size,
                           m->seg_dim, m->seg_dim + m->ver_dim, b, h, w, m->out_nhwc, s);
    case ST_SCORE:
        return launch_head3x3(B[m->bFeat], m->feat_c, m->w[st.slot], m->bias[st.slot], out_nchw, b, h8, w8, s);
    }
    return PVNET_E_INVALID;
}
}  // namespace

extern "C" {

int pvnet_backbone_num_stages(void) { return (int)resnet18_plan().stages.size(); }

const char *pvnet_backbone_stage_name(int stage)
{
    const pvnet_backbone &r18 = resnet18_plan();
    return (stage >= 0 && stage < (int)r18.stages.size()) ? r18.stages[stage].name.c_str() : "";
}

int pvnet_backbone_handle_num_stages(const pvnet_backbone_t *m) { return m ? (int)m->stages.size() : -1; }

const char *pvnet_backbone_handle_stage_name(const pvnet_backbone_t *m, int stage)
{
    return (m && stage >= 0 && stage < (int)m->stages.size()) ? m->stages[stage].name.c_str() : "";
}

int pvnet_backbone_run_stage(pvnet_backbone_t *m, int stage, const float *image_nchw, int b, int h, int w,
                             float *out_nchw, void *mask_out, int mask_elem_size, void *workspace,
                             size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(m, "null handle");
    PV_CHECK_ARG(stage >= 0 && stage < (int)m->stages.size(), "stage %d out of range", stage);
    std::vector<float *> B;
    const ImageSrc img{image_nchw, 0, {0, 0, 0}, {1, 1, 1}};
    int rc = prepare(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, &B);
    if (rc) return rc;
    return run_stage(m, m->stages[stage], B, img, b, h, w, out_nchw, mask_out, mask_elem_size, (cudaStream_t)stream);
}

static int forward_impl(pvnet_backbone_t *m, const ImageSrc &img, int b, int h, int w, float *out_nchw, void *mask_out,
                        int mask_elem_size, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    std::vector<float *> B;
    int rc = prepare(m, img, b, h, w, out_nchw, mask_out, mask_elem_size, workspace, workspace_bytes, &B);
    if (rc) return rc;
    for (const Stage &st : m->stages)
        if ((rc = run_stage(m, st, B, img, b, h, w, out_nchw, mask_out, mask_elem_size, (cudaStream_t)stream)))
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
