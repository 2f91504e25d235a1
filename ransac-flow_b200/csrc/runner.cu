// rf_run_layers: a whole conv network (ResNet-50 conv1..layer3, FeatureExtractor, the flow / matchability heads)
// executed from ONE host call: the layer list is walked here, in C++, so the per-layer cost on the host is a
// kernel launch (a few microseconds) instead of a Python -> ctypes round trip.
#include "common.cuh"

using namespace rf;

int rf_im2col_impl(const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, int Kpad, int round_out,
                   float* y, void* stream);
int rf_poolblur_impl(const float* x, int nimg, const int* hw_host, int C, int round_out, float* y, void* stream);
int rf_im2col_f16_impl(const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, int Kpad, void* y_f16, void* stream);
int rf_maxpool_f16_impl(const void* x_f16, int nimg, const int* hw_host, int C, int k, int stride, int pad, void* y_f16, void* stream);
int rf_stem7_f16_impl(const float* x, int nimg, const int* hw_host, const void* w_f16, const float* bias, int pool, void* y_f16, void* stream);
int rf_blur_f16_impl(const void* x_f16, int nimg, const int* hw_host, int C, int stride, void* y_f16, void* stream);
int rf_poolblur_f16_impl(const void* x_f16, int nimg, const int* hw_host, int C, void* y_f16, void* stream);
int rf_stem7_split_impl(const float* x, int nimg, const int* hw_host, const void* w_split, const float* bias, int pool, void* y_split, void* stream);
int rf_blur_split_impl(const void* x, int nimg, const int* hw_host, int C, int stride, void* y, void* stream);
int rf_poolblur_split_impl(const void* x, int nimg, const int* hw_host, int C, void* y, void* stream);
int rf_maxpool_split_impl(const void* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, void* y, void* stream);
int rf_im2col_split_impl(const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, int Kpad, void* y, void* stream);
int rf_blur_downsample_impl(const float* x, int nimg, const int* hw_host, int C, int stride, int round_out, float* y, void* stream);
int rf_stem3_split_impl(const float* x, int nimg, const int* hw_host, const float* w, const float* bias, void* y, void* stream);
int rf_conv2d_nhwc_dil(const float* x, int nimg, const int* hw_host, int Cin, const float* w, const float* w_tc, const float* bias,
                       const float* residual, int Cout, int R, int S, int stride, int pad, int dil, int relu, int engine, float* y, void* stream);

extern "C" int rf_run_layers(const rf_layer_t* L, int n, void* const* slots, int nimg, const int* hw_host, int engine, void* stream) {
    RF_REQUIRE(L != nullptr && n >= 1 && nimg >= 1 && nimg <= RF_MAX_IMGS, "rf_run_layers: bad arguments");
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
        RF_REQUIRE(dil == 1 || (l.op == RF_OP_CONV && engine == RF_ENGINE_SPLIT && !(l.flags & RF_LAYER_OUT_F32) && k == 3 && stride == 1),
                   "rf_run_layers: dilation is for RF_OP_CONV 3x3 / stride 1 layers with split outputs on engine 4");
        if (l.op == RF_OP_STEM7) {
            RF_REQUIRE(engine == RF_ENGINE_SPLIT || engine == RF_ENGINE_F16, "rf_run_layers: RF_OP_STEM7 needs engine 2 or 4");
            RF_REQUIRE(l.src == L[0].src && l.Cin == 3 && l.Cout == 64 && k == 7 && stride == 2 && pad == 3 && l.relu,
                       "rf_run_layers: RF_OP_STEM7 is the ResNet-50 stem on the fp32 input slot");
            const bool pool = (l.flags & RF_LAYER_STEM_POOL) != 0;
            const rf_layer_t* mp = pool && li + 1 < n ? &L[li + 1] : nullptr;
            RF_REQUIRE(!pool || (mp != nullptr && mp->op == RF_OP_MAXPOOL && mp->src == l.dst && mp->Cin == 64 && mp->k == 3 && mp->stride == 2 &&
                                 mp->pad == 1 && mp->dst >= 0 && mp->dst < RF_MAX_SLOTS && mp->dst != l.src),
                       "rf_run_layers: RF_LAYER_STEM_POOL needs the next layer to be a 3x3 / stride 2 / pad 1 max-pool of the stem's output");
            void* out = pool ? slots[mp->dst] : y;
            rc = engine == RF_ENGINE_SPLIT ? rf_stem7_split_impl(x, nimg, shw, l.w_f16, l.bias, pool, out, stream)
                                           : rf_stem7_f16_impl(x, nimg, shw, l.w_f16, l.bias, pool, out, stream);
            if (rc) return rc;
            if (pool) {         // the stem's own slot is never written: the pair's output is the max-pool's
                for (int i = 0; i < nimg; ++i)
                    for (int d = 0; d < 2; ++d) hw[mp->dst][2 * i + d] = ((shw[2 * i + d] - 1) / 2 + 1 - 1) / 2 + 1;
                known[mp->dst] = true;
                ++li;
                continue;
            }
        } else if (engine == RF_ENGINE_SPLIT) {
            // split activations ([2][P][C] fp16): the fp32 input image may only feed the stem; RF_LAYER_OUT_F32 convs write fp32
            if (l.op == RF_OP_CONV) {
                const float* res = l.res >= 0 ? static_cast<const float*>(slots[l.res]) : nullptr;
                rc = rf_conv2d_nhwc_dil(x, nimg, shw, l.Cin, l.w, static_cast<const float*>(l.w_f16), l.bias, res, l.Cout, k, k, stride, pad, dil,
                                        l.relu, (l.flags & RF_LAYER_OUT_F32) ? RF_ENGINE_SPLIT_OUT32 : RF_ENGINE_SPLIT, y, stream);
            } else if (l.op == RF_OP_CONV_DUAL) {
                RF_REQUIRE(l.src2 >= 0 && l.src2 < RF_MAX_SLOTS && known[l.src2] && l.dst != l.src2 && l.res < 0 && k == 1 && stride == 1 && pad == 0,
                           "rf_run_layers: RF_OP_CONV_DUAL needs a written second input slot, k = 1, stride 1, pad 0, no residual");
                rc = rf_conv1x1_dual_split(x, slots[l.src2], nimg, shw, hw[l.src2], l.Cin, l.Cin2, l.stride2, l.w_f16, l.bias, l.Cout, l.relu, y, stream);
            } else if (l.op == RF_OP_MAXPOOL) {
                rc = rf_maxpool_split_impl(x, nimg, shw, l.Cin, k, stride, pad, y, stream);
            } else if (l.op == RF_OP_BLUR) {
                k = 3; pad = 1;
                rc = rf_blur_split_impl(x, nimg, shw, l.Cin, stride, y, stream);
            } else if (l.op == RF_OP_POOLBLUR) {
                k = 4; stride = 2; pad = 1;
                rc = rf_poolblur_split_impl(x, nimg, shw, l.Cin, y, stream);
            } else if (l.op == RF_OP_IM2COL) {
                RF_REQUIRE(l.src == L[0].src, "rf_run_layers (engine 4): im2col reads the fp32 input slot");
                rc = rf_im2col_split_impl(x, nimg, shw, l.Cin, k, stride, pad, l.Cout, y, stream);
            } else if (l.op == RF_OP_STEM3) {
                RF_REQUIRE(l.src == L[0].src && l.Cin == 3 && l.Cout == 64 && k == 3 && stride == 2 && pad == 1 && l.relu,
                           "rf_run_layers: RF_OP_STEM3 is segNet's 3x3 / stride 2 / pad 1, 3 -> 64 stem conv (+ ReLU) on the fp32 input slot");
                rc = rf_stem3_split_impl(x, nimg, shw, l.w, l.bias, y, stream);
            } else {
                return fail_msg("rf_run_layers: unknown op");
            }
        } else if (engine == RF_ENGINE_F16) {
            // fp16 activations: the (fp32) input image may only feed the stem's im2col; everything after it is fp16
            if (l.op == RF_OP_CONV) {
                const float* res = l.res >= 0 ? static_cast<const float*>(slots[l.res]) : nullptr;
                if (l.flags & RF_LAYER_TF32)          // fp32 in / out on the TF32 engine (SIMT for shapes it does not cover)
                    rc = rf_conv2d_nhwc(x, nimg, shw, l.Cin, l.w, l.w_tc, l.bias, res, l.Cout, k, k, stride, pad, l.relu, RF_ENGINE_TF32, y, stream);
                else
                    rc = rf_conv2d_nhwc(x, nimg, shw, l.Cin, l.w, static_cast<const float*>(l.w_f16), l.bias, res, l.Cout, k, k, stride, pad, l.relu,
                                        (l.flags & RF_LAYER_OUT_F32) ? RF_ENGINE_F16_OUT32 : RF_ENGINE_F16, y, stream);
            } else if (l.op == RF_OP_MAXPOOL) {
                rc = rf_maxpool_f16_impl(x, nimg, shw, l.Cin, k, stride, pad, y, stream);
            } else if (l.op == RF_OP_BLUR) {
                k = 3; pad = 1;
                rc = rf_blur_f16_impl(x, nimg, shw, l.Cin, stride, y, stream);
            } else if (l.op == RF_OP_POOLBLUR) {
                k = 4; stride = 2; pad = 1;
                rc = rf_poolblur_f16_impl(x, nimg, shw, l.Cin, y, stream);
            } else if (l.op == RF_OP_IM2COL) {
                RF_REQUIRE(l.src == L[0].src, "rf_run_layers (engine 2): im2col reads the fp32 input slot");
                rc = rf_im2col_f16_impl(x, nimg, shw, l.Cin, k, stride, pad, l.Cout, y, stream);
            } else {
                return fail_msg("rf_run_layers: unknown op");
            }
        } else if (l.op == RF_OP_CONV) {
            const float* res = l.res >= 0 ? static_cast<const float*>(slots[l.res]) : nullptr;
            rc = rf_conv2d_nhwc(x, nimg, shw, l.Cin, l.w, l.w_tc, l.bias, res, l.Cout, k, k, stride, pad, l.relu, engine, y, stream);
        } else if (l.op == RF_OP_MAXPOOL) {
            rc = rf_maxpool2d_nhwc(x, nimg, shw, l.Cin, k, stride, pad, y, stream);
        } else if (l.op == RF_OP_BLUR) {
            k = 3; pad = 1;
            rc = rf_blur_downsample_impl(x, nimg, shw, l.Cin, stride, engine == 1 ? 1 : 0, y, stream);
        } else if (l.op == RF_OP_POOLBLUR) {
            k = 4; stride = 2; pad = 1;                 // size rule of maxpool(2,1) followed by blur(3, stride 2, pad 1)
            rc = rf_poolblur_impl(x, nimg, shw, l.Cin, engine == 1 ? 1 : 0, y, stream);
        } else if (l.op == RF_OP_IM2COL) {
            rc = rf_im2col_impl(x, nimg, shw, l.Cin, k, stride, pad, l.Cout, engine == 1 ? 1 : 0, y, stream);
        } else {
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
