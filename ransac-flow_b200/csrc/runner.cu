// rf_run_layers: a whole conv network (ResNet-50 conv1..layer3, FeatureExtractor, the flow / matchability heads)
// executed from ONE host call: the layer list is walked here, in C++, so the per-layer cost on the host is a
// kernel launch (a few microseconds) instead of a Python -> ctypes round trip.
#include "common.cuh"

using namespace rf;

int rf_maxpool(ActFormat f, const void* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, void* y, void* stream);
int rf_blur(ActFormat f, const void* x, int nimg, const int* hw_host, int C, int stride, void* y, void* stream);
int rf_poolblur(ActFormat f, const void* x, int nimg, const int* hw_host, int C, void* y, void* stream);
int rf_im2col(ActFormat f, const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, int Kpad, void* y, void* stream);
int rf_stem(ActFormat f, const float* x, int nimg, const int* hw_host, int k, int stride, const void* w, const float* bias, int pool, void* y,
            void* stream);
int rf_stem3(const float* x, int nimg, const int* hw_host, const float* w, const float* bias, void* y, void* stream);
int rf_conv2d_nhwc_dil(const float* x, int nimg, const int* hw_host, int Cin, const float* w, const float* w_tc, const float* bias,
                       const float* residual, int Cout, int R, int S, int stride, int pad, int dil, int relu, int engine, float* y, void* stream);

extern "C" int rf_run_layers(const rf_layer_t* L, int n, void* const* slots, int nimg, const int* hw_host, int engine, void* stream) {
    RF_REQUIRE(L != nullptr && n >= 1 && nimg >= 1 && nimg <= RF_MAX_IMGS, "rf_run_layers: bad arguments");
    const ActFormat f = act_format(engine);
    RF_REQUIRE(f != ACT_NONE, "rf_run_layers: layer programs run on engine 0 (fp32), 1 (TF32), 2 (fp16) or 4 (split)");
    static thread_local int hw[RF_MAX_SLOTS][2 * RF_MAX_IMGS];
    bool known[RF_MAX_SLOTS] = {false};
    RF_REQUIRE(L[0].src >= 0 && L[0].src < RF_MAX_SLOTS, "rf_run_layers: bad input slot");
    for (int i = 0; i < 2 * nimg; ++i) hw[L[0].src][i] = hw_host[i];
    known[L[0].src] = true;
    for (int li = 0; li < n; ++li) {
        const rf_layer_t& l = L[li];
        RF_REQUIRE(l.src >= 0 && l.src < RF_MAX_SLOTS && l.dst >= 0 && l.dst < RF_MAX_SLOTS && l.res < RF_MAX_SLOTS, "rf_run_layers: slot index out of range");
        RF_REQUIRE(known[l.src], "rf_run_layers: layer reads a slot nothing has written");
        RF_REQUIRE(l.dst != l.src && l.dst != l.res, "rf_run_layers: in-place layers are not supported");
        const int* shw = hw[l.src];
        const float* x = static_cast<const float*>(slots[l.src]);
        float* y = static_cast<float*>(slots[l.dst]);
        int rc = 0;
        int k = l.k, stride = l.stride, pad = l.pad;
        const int dil = l.dil > 1 ? l.dil : 1;
        RF_REQUIRE(dil == 1 || (l.op == RF_OP_CONV && f == ACT_SPLIT && !(l.flags & RF_LAYER_OUT_F32) && k == 3 && stride == 1),
                   "rf_run_layers: dilation is for RF_OP_CONV 3x3 / stride 1 layers with split outputs on engine 4");
        switch (l.op) {
        case RF_OP_CONV: {
            // split: 4 / 5 (RF_LAYER_OUT_F32); fp16: 2 / 3, or TF32 on fp32 slots (RF_LAYER_TF32); fp32 / TF32: the engine itself
            const bool out32 = (l.flags & RF_LAYER_OUT_F32) != 0;
            const int conv_engine = f == ACT_SPLIT ? (out32 ? RF_ENGINE_SPLIT_OUT32 : RF_ENGINE_SPLIT)
                                    : f == ACT_F16 ? ((l.flags & RF_LAYER_TF32) ? RF_ENGINE_TF32 : out32 ? RF_ENGINE_F16_OUT32 : RF_ENGINE_F16)
                                                   : engine;
            const float* w_tc = conv_engine >= RF_ENGINE_F16 ? static_cast<const float*>(l.w_f16) : l.w_tc;
            const float* res = l.res >= 0 ? static_cast<const float*>(slots[l.res]) : nullptr;
            rc = rf_conv2d_nhwc_dil(x, nimg, shw, l.Cin, l.w, w_tc, l.bias, res, l.Cout, k, k, stride, pad, dil, l.relu, conv_engine, y, stream);
            break;
        }
        case RF_OP_CONV_DUAL:
            RF_REQUIRE(f == ACT_SPLIT, "rf_run_layers: RF_OP_CONV_DUAL needs engine 4");
            RF_REQUIRE(l.src2 >= 0 && l.src2 < RF_MAX_SLOTS && known[l.src2] && l.dst != l.src2 && l.res < 0 && k == 1 && stride == 1 && pad == 0,
                       "rf_run_layers: RF_OP_CONV_DUAL needs a written second input slot, k = 1, stride 1, pad 0, no residual");
            rc = rf_conv1x1_dual_split(x, slots[l.src2], nimg, shw, hw[l.src2], l.Cin, l.Cin2, l.stride2, l.w_f16, l.bias, l.Cout, l.relu, y, stream);
            break;
        case RF_OP_STEM3:
            RF_REQUIRE(f == ACT_SPLIT, "rf_run_layers: RF_OP_STEM3 needs engine 4");
            RF_REQUIRE(l.src == L[0].src && l.Cin == 3 && l.Cout == 64 && k == 3 && stride == 2 && pad == 1 && l.relu,
                       "rf_run_layers: RF_OP_STEM3 is segNet's 3x3 / stride 2 / pad 1, 3 -> 64 stem conv (+ ReLU) on the fp32 input slot");
            rc = rf_stem3(x, nimg, shw, l.w, l.bias, y, stream);
            break;
        case RF_OP_STEM7: {
            RF_REQUIRE(f == ACT_F16 || f == ACT_SPLIT, "rf_run_layers: RF_OP_STEM7 needs engine 2 or 4");
            RF_REQUIRE(l.src == L[0].src && l.Cin == 3 && l.Cout == 64 && ((k == 7 && stride == 2 && pad == 3) || (k == 3 && stride == 1 && pad == 1)) && l.relu,
                       "rf_run_layers: RF_OP_STEM7 is the ResNet-50 stem (7x7 / 2 / pad 3) or the FeatureExtractor stem (3x3 / 1 / pad 1) on the fp32 input slot");
            const bool pool = (l.flags & RF_LAYER_STEM_POOL) != 0;
            RF_REQUIRE(!pool || k == 7, "rf_run_layers: RF_LAYER_STEM_POOL pools the 7x7 stem");
            const rf_layer_t* mp = pool && li + 1 < n ? &L[li + 1] : nullptr;
            RF_REQUIRE(!pool || (mp != nullptr && mp->op == RF_OP_MAXPOOL && mp->src == l.dst && mp->Cin == 64 && mp->k == 3 && mp->stride == 2 &&
                                 mp->pad == 1 && mp->dst >= 0 && mp->dst < RF_MAX_SLOTS && mp->dst != l.src),
                       "rf_run_layers: RF_LAYER_STEM_POOL needs the next layer to be a 3x3 / stride 2 / pad 1 max-pool of the stem's output");
            rc = rf_stem(f, x, nimg, shw, k, stride, l.w_f16, l.bias, pool, pool ? slots[mp->dst] : y, stream);
            if (rc) return rc;
            if (pool) {         // the stem's own slot is never written: the pair's output is the max-pool's
                for (int i = 0; i < nimg; ++i)
                    for (int d = 0; d < 2; ++d) hw[mp->dst][2 * i + d] = ((shw[2 * i + d] - 1) / 2 + 1 - 1) / 2 + 1;
                known[mp->dst] = true;
                ++li;
                continue;
            }
            break;
        }
        case RF_OP_MAXPOOL:
            rc = rf_maxpool(f, x, nimg, shw, l.Cin, k, stride, pad, y, stream);
            break;
        case RF_OP_BLUR:
            k = 3; pad = 1;
            rc = rf_blur(f, x, nimg, shw, l.Cin, stride, y, stream);
            break;
        case RF_OP_POOLBLUR:
            k = 4; stride = 2; pad = 1;                 // size rule of maxpool(2,1) followed by blur(3, stride 2, pad 1)
            rc = rf_poolblur(f, x, nimg, shw, l.Cin, y, stream);
            break;
        case RF_OP_IM2COL:
            RF_REQUIRE(l.src == L[0].src, "rf_run_layers: im2col reads the fp32 input slot");
            rc = rf_im2col(f, x, nimg, shw, l.Cin, k, stride, pad, l.Cout, y, stream);
            break;
        default:
            return fail_msg("rf_run_layers: unknown op");
        }
        if (rc) return rc;
        for (int i = 0; i < nimg; ++i) {
            hw[l.dst][2 * i] = (shw[2 * i] + 2 * pad - dil * (k - 1) - 1) / stride + 1;
            hw[l.dst][2 * i + 1] = (shw[2 * i + 1] + 2 * pad - dil * (k - 1) - 1) / stride + 1;
        }
        known[l.dst] = true;
    }
    return 0;
}
