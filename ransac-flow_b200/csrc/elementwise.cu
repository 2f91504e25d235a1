// HBM-bound kernels of the hot path: pooling, anti-aliased downsampling, L2
// normalisation, local correlation, flow/matchability heads' epilogues, image
// pre-processing, homography grids, bilinear sampling and the fused
// fine-flow composition.  All NHWC fp32, coalesced along channels, vectorised
// (float4) where the channel count allows.
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"

namespace rf {

// 16-byte vectors of the activation type: 4 floats or 8 halves; arithmetic is always fp32.  The kernels of the layer ops
// (max-pool, im2col, blur, pool + blur, L2 normalisation) are written once over Vec16<T>, T = float, __half or SplitH.
template <typename T> struct Vec16;
template <> struct Vec16<float> {
    typedef float elem;
    static constexpr int N = 4;
    static __device__ __forceinline__ void load(const float* p, long long, float (&v)[4]) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void store(float* p, long long, const float (&v)[4], int round_out) {
        float4 t = make_float4(v[0], v[1], v[2], v[3]);
        if (round_out) { t.x = round_tf32(t.x); t.y = round_tf32(t.y); t.z = round_tf32(t.z); t.w = round_tf32(t.w); }
        *reinterpret_cast<float4*>(p) = t;
    }
};
template <> struct Vec16<__half> {
    typedef __half elem;
    static constexpr int N = 8;
    static __device__ __forceinline__ void load(const __half* p, long long, float (&v)[8]) {
        const uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
        const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
    }
    static __device__ __forceinline__ void store(__half* p, long long, const float (&v)[8], int) {
        uint4 t;
        __half2* h = reinterpret_cast<__half2*>(&t);
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
        *reinterpret_cast<uint4*>(p) = t;
    }
};
// engine 4: split tensors, two fp16 planes `plane` elements apart (x = hi + lo * 2^-11); values are rebuilt exactly in fp32,
// results are split again (split_store8, common.cuh)
struct SplitH {};
__device__ __forceinline__ void split_load8(const __half* p, long long plane, float (&v)[8]) {
    const uint4 th = __ldg(reinterpret_cast<const uint4*>(p)), tl = __ldg(reinterpret_cast<const uint4*>(p + plane));
    const __half2* h = reinterpret_cast<const __half2*>(&th);
    const __half2* l = reinterpret_cast<const __half2*>(&tl);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 fh = __half22float2(h[e]), fl = __half22float2(l[e]);
        v[2 * e] = fmaf(fl.x, 0.00048828125f, fh.x);
        v[2 * e + 1] = fmaf(fl.y, 0.00048828125f, fh.y);
    }
}
template <> struct Vec16<SplitH> {
    typedef __half elem;
    static constexpr int N = 8;
    static __device__ __forceinline__ void load(const __half* p, long long plane, float (&v)[8]) { split_load8(p, plane, v); }
    static __device__ __forceinline__ void store(__half* p, long long plane, const float (&v)[8], int) { split_store8(p, plane, v); }
};

// ---------------------------------------------------------------------------
// nn.MaxPool2d(k, stride, pad) on a ragged NHWC batch (model/model.py:71: k=2,s=1; torchvision resnet: k=3,s=2,p=1).  One
// thread per (output pixel, 16-byte vector).
// ---------------------------------------------------------------------------
// running maximum of 16-byte vectors, from -inf: fp32 values (split: rebuilt, and split again on the store) ...
template <typename T> struct VecMax {
    float m[Vec16<T>::N];
    __device__ __forceinline__ VecMax() {
#pragma unroll
        for (int e = 0; e < Vec16<T>::N; ++e) m[e] = -INFINITY;
    }
    __device__ __forceinline__ void add(const typename Vec16<T>::elem* p, long long plane) {
        float v[Vec16<T>::N];
        Vec16<T>::load(p, plane, v);
#pragma unroll
        for (int e = 0; e < Vec16<T>::N; ++e) m[e] = fmaxf(m[e], v[e]);
    }
    __device__ __forceinline__ void store(typename Vec16<T>::elem* p, long long plane) const { Vec16<T>::store(p, plane, m, 0); }
};
// ... fp16: the packed halves with __hmax2 (half the registers of eight fp32 values)
template <> struct VecMax<__half> {
    __half2 m[4];
    __device__ __forceinline__ VecMax() {
#pragma unroll
        for (int e = 0; e < 4; ++e) m[e] = __float2half2_rn(-INFINITY);
    }
    __device__ __forceinline__ void add(const __half* p, long long) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) m[e] = __hmax2(m[e], h[e]);
    }
    __device__ __forceinline__ void store(__half* p, long long) const {
        uint4 o;
        __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = m[e];
        *reinterpret_cast<uint4*>(p) = o;
    }
};

template <typename T>
__global__ void maxpool_kernel(const __grid_constant__ ImgSet set, const typename Vec16<T>::elem* __restrict__ x, typename Vec16<T>::elem* __restrict__ y,
                               int C, int k, int stride, int pad, long long pin, long long pout) {
    constexpr int VN = Vec16<T>::N;
    const int cvn = C / VN;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = set.out_pix[set.n] * cvn;
    if (t >= total) return;
    long long pm = t / cvn;
    int cv = (int)(t - pm * cvn);
    int im = find_img(set, pm);
    int local = (int)(pm - set.out_pix[im]);
    int oy = local / set.Wo[im], ox = local - oy * set.Wo[im];
    const int H = set.H[im], W = set.W[im];
    VecMax<T> m;
    for (int r = 0; r < k; ++r) {
        int iy = oy * stride - pad + r;
        if (iy < 0 || iy >= H) continue;
        for (int s = 0; s < k; ++s) {
            int ix = ox * stride - pad + s;
            if (ix < 0 || ix >= W) continue;
            m.add(x + (set.in_pix[im] + (long long)iy * W + ix) * C + cv * VN, pin);
        }
    }
    m.store(y + pm * C + cv * VN, pout);
}

// ---------------------------------------------------------------------------
// im2col for the few-channel stems (3 -> 64): row p of the output holds the k*k*C patch of output pixel p in
// (r, s, c) order, zero padded to Kpad (a multiple of 32 floats = one 128-byte swizzle row), so that the stem
// becomes a 1x1 convolution the tensor-core engine can read with TMA.  One thread per (pixel, patch element).
// ---------------------------------------------------------------------------
// grid: (ceil(Ho*Wo*Kpad/4 / 256), image); one thread per float4 of the output; 32-bit index math.
template <int KC, int CC, int KPADC>      // compile-time (k, C, Kpad) for the two stems (0 = runtime values)
__global__ void im2col_kernel(const __grid_constant__ ImgSet set, const float* __restrict__ x, float* __restrict__ y,
                              int C_, int k_, int stride, int pad, int Kpad_, int round_out) {
    const int C = CC ? CC : C_, k = KC ? KC : k_, Kpad = KPADC ? KPADC : Kpad_;
    const int im = blockIdx.y;
    const int q4 = Kpad >> 2;                                   // float4 per output row
    const int Wo = set.Wo[im], H = set.H[im], W = set.W[im];
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned total = (unsigned)(set.Ho[im] * Wo) * (unsigned)q4;
    if (idx >= total) return;
    const unsigned local = idx / (unsigned)q4;
    const int e0 = (int)(idx - local * (unsigned)q4) * 4;
    const int oy = (int)(local / (unsigned)Wo), ox = (int)(local - (unsigned)oy * (unsigned)Wo);
    const int kkc = k * k * C, kc = k * C;
    const float* src = x + set.in_pix[im] * C;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int e = e0 + j;
        float t = 0.f;
        if (e < kkc) {
            const int r = e / kc, rem = e - r * kc;             // (r, s, c) order: rem = s*C + c is contiguous in the input row
            const int iy = oy * stride - pad + r;
            const int ixc = (ox * stride - pad) * C + rem;      // element offset inside the input row
            if (iy >= 0 && iy < H && ixc >= 0 && ixc < W * C) t = __ldg(src + (long long)iy * W * C + ixc);
            if (round_out) t = round_tf32(t);
        }
        v[j] = t;
    }
    reinterpret_cast<float4*>(y + (set.out_pix[im] + local) * Kpad)[e0 >> 2] = make_float4(v[0], v[1], v[2], v[3]);
}

// ---------------------------------------------------------------------------
// model/downsample.py:12-46: ReflectionPad2d(1) + depthwise [1 2 1]x[1 2 1]/16, stride s
// ---------------------------------------------------------------------------
__device__ __forceinline__ int reflect1(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

template <typename T>
__global__ void blur_kernel(const __grid_constant__ ImgSet set, const typename Vec16<T>::elem* __restrict__ x, typename Vec16<T>::elem* __restrict__ y,
                            int C, int stride, int round_out, long long pin = 0, long long pout = 0) {
    constexpr int VN = Vec16<T>::N;
    const int cvn = C / VN;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = set.out_pix[set.n] * cvn;
    if (t >= total) return;
    long long pm = t / cvn;
    int cv = (int)(t - pm * cvn);
    int im = find_img(set, pm);
    int local = (int)(pm - set.out_pix[im]);
    int oy = local / set.Wo[im], ox = local - oy * set.Wo[im];
    const int H = set.H[im], W = set.W[im];
    float acc[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) acc[e] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        int iy = reflect1(oy * stride - 1 + r, H);
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            int ix = reflect1(ox * stride - 1 + s, W);
            float wgt = ((r == 1) ? 2.f : 1.f) * ((s == 1) ? 2.f : 1.f) * 0.0625f;
            float v[VN];
            Vec16<T>::load(x + (set.in_pix[im] + (long long)iy * W + ix) * C + cv * VN, pin, v);
#pragma unroll
            for (int e = 0; e < VN; ++e) acc[e] = fmaf(wgt, v[e], acc[e]);
        }
    }
    Vec16<T>::store(y + pm * C + cv * VN, pout, acc, round_out);
}

// ---------------------------------------------------------------------------
// FeatureExtractor stem tail fused (model/model.py:71-72): MaxPool2d(2, stride 1) followed by the anti-aliased
// stride-2 blur (reflect-pad 1, [1 2 1]^2/16).  The (H-1) x (W-1) pooled map is never written: each output reads
// the 4 x 4 input window its 3 x 3 pooled neighbourhood covers (78.6 MB in, 19.7 MB out at 480x640 instead of
// 78.6 + 78.6 + 78.6 + 19.7).
// ---------------------------------------------------------------------------
template <typename T>
__global__ void poolblur_kernel(const __grid_constant__ ImgSet set, const typename Vec16<T>::elem* __restrict__ x, typename Vec16<T>::elem* __restrict__ y,
                                int C, int round_out, long long pin = 0, long long pout = 0) {
    constexpr int VN = Vec16<T>::N;
    const int cvn = C / VN;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = set.out_pix[set.n] * cvn;
    if (t >= total) return;
    long long pm = t / cvn;
    int cv = (int)(t - pm * cvn);
    int im = find_img(set, pm);
    int local = (int)(pm - set.out_pix[im]);
    int oy = local / set.Wo[im], ox = local - oy * set.Wo[im];
    const int H = set.H[im], W = set.W[im];
    const int Hp = H - 1, Wp = W - 1;                       // pooled map size
    const typename Vec16<T>::elem* base = x + set.in_pix[im] * C + cv * VN;
    float acc[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) acc[e] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int py = reflect1(oy * 2 - 1 + r, Hp);
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            const int px = reflect1(ox * 2 - 1 + s, Wp);
            const float wgt = ((r == 1) ? 2.f : 1.f) * ((s == 1) ? 2.f : 1.f) * 0.0625f;
            float a[VN], b[VN], c[VN], d[VN];
            Vec16<T>::load(base + ((long long)py * W + px) * C, pin, a);
            Vec16<T>::load(base + ((long long)py * W + px + 1) * C, pin, b);
            Vec16<T>::load(base + ((long long)(py + 1) * W + px) * C, pin, c);
            Vec16<T>::load(base + ((long long)(py + 1) * W + px + 1) * C, pin, d);
#pragma unroll
            for (int e = 0; e < VN; ++e) acc[e] = fmaf(wgt, fmaxf(fmaxf(a[e], b[e]), fmaxf(c[e], d[e])), acc[e]);
        }
    }
    Vec16<T>::store(y + pm * C + cv * VN, pout, acc, round_out);
}

// ---------------------------------------------------------------------------
// F.normalize(dim=1): one warp per pixel (coarseAlignFeatMatch.py:106,124; evaluation.py:26,184); fp32 arithmetic and
// output whatever the input format.  `y` (nullable when the planes are written): the fp32 rows.  Split input only, `yhi` /
// `ylo` (nullable): ALSO the normalised rows as the fp16 hi / lo * 2^11 planes the fp16-split correlation kernel reads
// (rf_corr_mutual_nn with presplit operands), which saves its split pass.
// ---------------------------------------------------------------------------
template <typename T>
__global__ void l2norm_kernel(const typename Vec16<T>::elem* __restrict__ x, long long plane, long long P, int C,
                              const unsigned char* __restrict__ mask, float* __restrict__ y, __half* __restrict__ yhi, __half* __restrict__ ylo) {
    constexpr int VN = Vec16<T>::N;
    constexpr bool planes = std::is_same<T, SplitH>::value;
    long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (pix >= P) return;
    const typename Vec16<T>::elem* src = x + pix * C;
    float4* dst = reinterpret_cast<float4*>(y + pix * C);
    const int cvn = C / VN;
    if (mask != nullptr && mask[pix] == 0) {
        if (y != nullptr)
            for (int c = lane; c < C / 4; c += 32) dst[c] = make_float4(0, 0, 0, 0);
        if constexpr (planes)
            if (yhi != nullptr)
                for (int c = lane; c < cvn; c += 32) {
                    reinterpret_cast<uint4*>(yhi + pix * C)[c] = make_uint4(0, 0, 0, 0);
                    reinterpret_cast<uint4*>(ylo + pix * C)[c] = make_uint4(0, 0, 0, 0);
                }
        return;
    }
    // (a single-pass variant that keeps the row in registers measured slower: 72 vs 55 us for the three calls of a pair)
    float ss = 0.f;
    for (int c = lane; c < cvn; c += 32) {
        float v[VN];
        Vec16<T>::load(src + c * VN, plane, v);
#pragma unroll
        for (int e = 0; e < VN; ++e) ss = fmaf(v[e], v[e], ss);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
    float denom = fmaxf(sqrtf(ss), 1e-12f);
    for (int c = lane; c < cvn; c += 32) {
        float v[VN];
        Vec16<T>::load(src + c * VN, plane, v);
#pragma unroll
        for (int e = 0; e < VN; ++e) v[e] = __fdiv_rn(v[e], denom);
        if (y != nullptr)
#pragma unroll
            for (int q = 0; q < VN / 4; ++q) dst[c * (VN / 4) + q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        if constexpr (planes)
            if (yhi != nullptr) split_store8(yhi + pix * C + c * 8, (ylo - yhi), v);
    }
}

// ---------------------------------------------------------------------------
// model/model.py:129-160 CorrNeigh: out[n,r,c,i*k+j] = sum_ch x[n,r,c,ch] * y[n,r+i-k/2,c+j-k/2,ch]
// one warp per output pixel, lanes over channels, k*k shuffled reductions
// ---------------------------------------------------------------------------
// `out2` (nullable): ALSO write CorrNeigh(y, x) there.  corr21[p][d] = <y_p, x_(p+d)> = <x_(p+d), y_p> = corr12[p+d][-d], the
// same dot product (fmaf(a, b, acc) with a and b swapped is the same operation, so the bits are equal): the warp of
// pixel p scatters every in-image tap to corr21[p+d][-d] and writes the zero of its own out-of-image taps, which covers
// every entry of corr21 exactly once.  One launch instead of two (evaluation/evalHpatch/evaluation.py:29-30).
// round_out: 0 fp32, 1 fp32 rounded to TF32, 2 fp16, 3 split (engine 4: [2][rows][ldo] fp16 planes).  Mode 3 with `out2`: `out` is
// the standalone corr12 tensor (planes P * ldo apart) and `out2` the two-image tensor [corr12 ; corr21] (2P rows, planes
// 2P * ldo apart) the matchability head runs on - corr12 is written to both.
__device__ __forceinline__ void corr_store(float* out, long long idx, float v, int round_out, long long plane) {
    if (round_out == 3) {
        const float a = fminf(fmaxf(v, -65504.f), 65504.f);
        const __half h = __float2half_rn(a);
        reinterpret_cast<__half*>(out)[idx] = h;
        reinterpret_cast<__half*>(out)[idx + plane] = __float2half_rn((a - __half2float(h)) * 2048.f);
    } else if (round_out == 2) {
        reinterpret_cast<__half*>(out)[idx] = __float2half_rn(v);
    } else {
        out[idx] = round_out ? round_tf32(v) : v;
    }
}

__global__ void corr_neigh_kernel(const float* __restrict__ x, const float* __restrict__ y, int N, int h, int w, int C, int k, int ldo, int round_out,
                                  float* __restrict__ out, float* __restrict__ out2) {
    long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    long long P = (long long)N * h * w;
    if (pix >= P) return;
    int n = (int)(pix / ((long long)h * w));
    int rem = (int)(pix - (long long)n * h * w);
    int r = rem / w, c = rem - r * w;
    const int pad = k / 2, c4n = C >> 2;
    const bool split = round_out == 3;
    const long long plane1 = P * ldo, plane2 = 2 * P * ldo;                  // split planes of `out` / of the two-image `out2`
    const float4* xs = reinterpret_cast<const float4*>(x + pix * C);
    // C <= 1024: up to 8 float4 per lane kept in registers
    float4 xv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) xv[q] = (lane + 32 * q < c4n) ? __ldg(xs + lane + 32 * q) : make_float4(0, 0, 0, 0);
    for (int i = 0; i < k; ++i) {
        int yr = r + i - pad;
        for (int j = 0; j < k; ++j) {
            int yc = c + j - pad;
            float acc = 0.f;
            if (yr >= 0 && yr < h && yc >= 0 && yc < w) {
                const float4* ys = reinterpret_cast<const float4*>(y + (((long long)n * h + yr) * w + yc) * C);
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    if (lane + 32 * q < c4n) {
                        float4 v = __ldg(ys + lane + 32 * q);
                        acc = fmaf(xv[q].x, v.x, acc); acc = fmaf(xv[q].y, v.y, acc);
                        acc = fmaf(xv[q].z, v.z, acc); acc = fmaf(xv[q].w, v.w, acc);
                    }
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
            if (lane == 0) {
                corr_store(out, pix * ldo + i * k + j, acc, round_out, plane1);
                if (out2 != nullptr) {
                    if (split) corr_store(out2, pix * ldo + i * k + j, acc, 3, plane2);
                    const bool inside = yr >= 0 && yr < h && yc >= 0 && yc < w;
                    // inside: entry (p + d, -d) of the swapped volume; outside: this pixel's own (zero) entry (p, d)
                    const long long q = inside ? (((long long)n * h + yr) * w + yc) : pix;
                    const int e = inside ? (k - 1 - i) * k + (k - 1 - j) : i * k + j;
                    if (split) corr_store(out2, (P + q) * ldo + e, acc, 3, plane2);
                    else corr_store(out2, q * ldo + e, acc, round_out, 0);
                }
            }
        }
    }
    for (int cz = k * k + lane; cz < ldo; cz += 32) {
        corr_store(out, pix * ldo + cz, 0.f, round_out, plane1);
        if (out2 != nullptr) {
            if (split) { corr_store(out2, pix * ldo + cz, 0.f, 3, plane2); corr_store(out2, (P + pix) * ldo + cz, 0.f, 3, plane2); }
            else corr_store(out2, pix * ldo + cz, 0.f, round_out, 0);
        }
    }
}

// k = 7 (every configuration of the reference): the 49 dot products of a pixel are accumulated per lane in registers and
// reduced with ONE multi-value butterfly (62 shuffles instead of 49 x 5): at each step a lane keeps half of its values and
// hands the other half to its partner, so lane L ends up with the complete sums 2L and 2L + 1 and the warp stores its 49
// (64 with padding) outputs as one coalesced row.  Eight warps of a CTA take eight horizontally adjacent pixels, whose
// 7 x 14 y-neighbourhood is mostly shared in L1.  Same products, same per-lane channel order and the same reduction tree for
// every tap, so CorrNeigh(y, x) written from here is bit-identical to a separate launch (see corr_neigh_kernel).
__global__ void __launch_bounds__(256)
corr_neigh7_kernel(const float* __restrict__ x, const float* __restrict__ y, int N, int h, int w, int C, int ldo, int round_out,
                   float* __restrict__ out, float* __restrict__ out2) {
    constexpr int K = 7, KK = 49, PAD = 3;
    const long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long P = (long long)N * h * w;
    if (pix >= P) return;
    const int n = (int)(pix / ((long long)h * w));
    const int rem = (int)(pix - (long long)n * h * w);
    const int r = rem / w, c = rem - r * w;
    const int c4n = C >> 2;
    const bool split = round_out == 3;
    const long long plane1 = P * ldo, plane2 = 2 * P * ldo;
    const float4* xs = reinterpret_cast<const float4*>(x + pix * C);
    float4 xv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) xv[q] = (lane + 32 * q < c4n) ? __ldg(xs + lane + 32 * q) : make_float4(0, 0, 0, 0);
    float a[64];
#pragma unroll
    for (int t = 0; t < 64; ++t) a[t] = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const int yr = r + i - PAD;
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const int yc = c + j - PAD;
            if (yr >= 0 && yr < h && yc >= 0 && yc < w) {
                const float4* ys = reinterpret_cast<const float4*>(y + (((long long)n * h + yr) * w + yc) * C);
                float acc = 0.f;
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    if (lane + 32 * q < c4n) {
                        const float4 v = __ldg(ys + lane + 32 * q);
                        acc = fmaf(xv[q].x, v.x, acc); acc = fmaf(xv[q].y, v.y, acc);
                        acc = fmaf(xv[q].z, v.z, acc); acc = fmaf(xv[q].w, v.w, acc);
                    }
                a[i * K + j] = acc;
            }
        }
    }
    // multi-value butterfly: 64 -> 32 -> 16 -> 8 -> 4 -> 2 values per lane
#pragma unroll
    for (int s = 16, nv = 32; s >= 1; s >>= 1, nv >>= 1) {
        const bool up = (lane & s) != 0;
#pragma unroll
        for (int v = 0; v < nv; ++v) {
            const float send = up ? a[v] : a[v + nv];
            const float keep = up ? a[v + nv] : a[v];
            a[v] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
    }
    // lane L holds taps 2L and 2L + 1 (taps >= 49 are the zero padding of a 64-wide row)
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int t = 2 * lane + u;
        if (t >= ldo) continue;
        const float v = a[u];
        corr_store(out, pix * ldo + t, v, round_out, plane1);
        if (out2 != nullptr) {
            if (split) corr_store(out2, pix * ldo + t, v, 3, plane2);
            if (t < KK) {
                const int i = t / K, j = t - i * K;
                const int yr = r + i - PAD, yc = c + j - PAD;
                const bool inside = yr >= 0 && yr < h && yc >= 0 && yc < w;
                const long long q = inside ? (((long long)n * h + yr) * w + yc) : pix;
                const int e = inside ? (KK - 1 - t) : t;
                if (split) corr_store(out2, (P + q) * ldo + e, v, 3, plane2);
                else corr_store(out2, q * ldo + e, v, round_out, 0);
            } else {
                if (split) corr_store(out2, (P + pix) * ldo + t, 0.f, 3, plane2);
                else corr_store(out2, pix * ldo + t, 0.f, round_out, 0);
            }
        }
    }
    for (int t = 64 + lane; t < ldo; t += 32) {          // ldo > 64: remaining zero columns
        corr_store(out, pix * ldo + t, 0.f, round_out, plane1);
        if (out2 != nullptr) {
            if (split) { corr_store(out2, pix * ldo + t, 0.f, 3, plane2); corr_store(out2, (P + pix) * ldo + t, 0.f, 3, plane2); }
            else corr_store(out2, pix * ldo + t, 0.f, round_out, 0);
        }
    }
}

// ---------------------------------------------------------------------------
// model/model.py:226-233: softmax over k*k channels + expected offset.  logits NHWC [P][k*k]
// ---------------------------------------------------------------------------
__global__ void softmax_flow_kernel(const float* __restrict__ logits, int N, int h, int w, int k, float* __restrict__ flow) {
    long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long hw = (long long)h * w;
    if (pix >= N * hw) return;
    const int kk = k * k, pad = k / 2;
    const float* l = logits + pix * kk;
    float m = -INFINITY;
    for (int q = 0; q < kk; ++q) m = fmaxf(m, __ldg(l + q));
    float sum = 0.f, sx = 0.f, sy = 0.f;
    for (int q = 0; q < kk; ++q) {
        float e = expf(__ldg(l + q) - m);
        sum += e;
        sx = fmaf(e, (float)(q % k - pad), sx);
        sy = fmaf(e, (float)(q / k - pad), sy);
    }
    int n = (int)(pix / hw);
    long long rem = pix - n * hw;
    // flowX = sum p*gridX / size(3) * 2 ; flowY = sum p*gridY / size(2) * 2
    flow[(n * 2 + 0) * hw + rem] = (sx / sum) / (float)w * 2.f;
    flow[(n * 2 + 1) * hw + rem] = (sy / sum) / (float)h * 2.f;
}

__global__ void sigmoid_kernel(const float* __restrict__ x, long long n, float* __restrict__ y) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = 1.f / (1.f + expf(-x[i]));
}

// ---------------------------------------------------------------------------
// torchvision ToTensor (+ Normalize): exact op order div(255), sub(mean), div(std)
// ---------------------------------------------------------------------------
__global__ void preproc_kernel(const unsigned char* __restrict__ img, long long n, int normalize, float* __restrict__ out) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = (int)(i % 3);
    float v = __fdiv_rn((float)img[i], 255.f);
    if (normalize) {
        const float mean = (c == 0) ? 0.485f : (c == 1 ? 0.456f : 0.406f);
        const float sd = (c == 0) ? 0.229f : (c == 1 ? 0.224f : 0.225f);
        v = __fdiv_rn(__fsub_rn(v, mean), sd);
    }
    out[i] = v;
}

// the same arithmetic, 12 bytes (4 RGB pixels) per thread: three 32-bit loads, three float4 stores
__device__ __forceinline__ float preproc_one(unsigned int byte, int c, int normalize) {
    float v = __fdiv_rn((float)byte, 255.f);
    if (normalize) {
        const float mean = (c == 0) ? 0.485f : (c == 1 ? 0.456f : 0.406f);
        const float sd = (c == 0) ? 0.229f : (c == 1 ? 0.224f : 0.225f);
        v = __fdiv_rn(__fsub_rn(v, mean), sd);
    }
    return v;
}
__global__ void preproc_vec_kernel(const unsigned int* __restrict__ img, long long ngroups, int normalize, float4* __restrict__ out) {
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    const unsigned int w0 = __ldg(img + 3 * g), w1 = __ldg(img + 3 * g + 1), w2 = __ldg(img + 3 * g + 2);
    // bytes 0..11 of the group: channel = byte index % 3 (a group starts on a pixel boundary)
    out[3 * g] = make_float4(preproc_one(w0 & 255u, 0, normalize), preproc_one((w0 >> 8) & 255u, 1, normalize),
                             preproc_one((w0 >> 16) & 255u, 2, normalize), preproc_one(w0 >> 24, 0, normalize));
    out[3 * g + 1] = make_float4(preproc_one(w1 & 255u, 1, normalize), preproc_one((w1 >> 8) & 255u, 2, normalize),
                                 preproc_one((w1 >> 16) & 255u, 0, normalize), preproc_one(w1 >> 24, 1, normalize));
    out[3 * g + 2] = make_float4(preproc_one(w2 & 255u, 2, normalize), preproc_one((w2 >> 8) & 255u, 0, normalize),
                                 preproc_one((w2 >> 16) & 255u, 1, normalize), preproc_one(w2 >> 24, 2, normalize));
}

// ---------------------------------------------------------------------------
// PIL ImagingResample (8 bits per channel, fixed point, one pass)
// ---------------------------------------------------------------------------
#define RF_PRECISION_BITS 22
__device__ __forceinline__ unsigned char clip8(int ss) {
    int v = ss >> RF_PRECISION_BITS;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}
// horizontal pass: one thread per output PIXEL (all channels), so the coefficient row is walked once
__global__ void resample_h_kernel(const unsigned char* __restrict__ in, int in_h, int in_w, int ch, const int* __restrict__ bounds,
                                  const int* __restrict__ kk, int ksize, int out_w, unsigned char* __restrict__ out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)in_h * out_w) return;
    const int ox = (int)(t % out_w), oy = (int)(t / out_w);
    const int lo = bounds[2 * ox], cnt = bounds[2 * ox + 1];
    const int* k = kk + (long long)ox * ksize;
    const unsigned char* row = in + ((long long)oy * in_w + lo) * ch;
    if (ch == 3) {
        int s0 = 1 << (RF_PRECISION_BITS - 1), s1 = s0, s2 = s0;
        for (int x = 0; x < cnt; ++x) {
            const int kx = __ldg(k + x);
            s0 += (int)row[3 * x] * kx; s1 += (int)row[3 * x + 1] * kx; s2 += (int)row[3 * x + 2] * kx;
        }
        unsigned char* o = out + t * 3;
        o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
    } else {
        for (int c = 0; c < ch; ++c) {
            int ss = 1 << (RF_PRECISION_BITS - 1);
            for (int x = 0; x < cnt; ++x) ss += (int)row[(long long)x * ch + c] * __ldg(k + x);
            out[t * ch + c] = clip8(ss);
        }
    }
}
// vertical pass: one thread per 4 consecutive bytes of an output row (rows are W*ch bytes, a multiple of 4 here)
__global__ void resample_v_kernel(const unsigned char* __restrict__ in, int in_h, int row_bytes, const int* __restrict__ bounds,
                                  const int* __restrict__ kk, int ksize, int out_h, unsigned char* __restrict__ out) {
    const int q = row_bytes >> 2;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)out_h * q) return;
    const int xq = (int)(t % q), oy = (int)(t / q);
    const int lo = bounds[2 * oy], cnt = bounds[2 * oy + 1];
    const int* k = kk + (long long)oy * ksize;
    const unsigned int* col = reinterpret_cast<const unsigned int*>(in + (long long)lo * row_bytes) + xq;
    int s0 = 1 << (RF_PRECISION_BITS - 1), s1 = s0, s2 = s0, s3 = s0;
    for (int y = 0; y < cnt; ++y) {
        const unsigned int v = __ldg(col + (long long)y * q);
        const int ky = __ldg(k + y);
        s0 += (int)(v & 0xFF) * ky; s1 += (int)((v >> 8) & 0xFF) * ky; s2 += (int)((v >> 16) & 0xFF) * ky; s3 += (int)(v >> 24) * ky;
    }
    reinterpret_cast<unsigned int*>(out)[t] = (unsigned)clip8(s0) | ((unsigned)clip8(s1) << 8) | ((unsigned)clip8(s2) << 16) | ((unsigned)clip8(s3) << 24);
}
// generic fallback (any row length / alignment): one thread per output byte
__global__ void resample_u8_kernel(const unsigned char* __restrict__ in, int in_h, int in_w, int ch, int horizontal,
                                   const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int out_size,
                                   unsigned char* __restrict__ out) {
    const int out_h = horizontal ? in_h : out_size, out_w = horizontal ? out_size : in_w;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = (long long)out_h * out_w * ch;
    if (t >= total) return;
    int c = (int)(t % ch);
    long long pq = t / ch;
    int ox = (int)(pq % out_w), oy = (int)(pq / out_w);
    int o = horizontal ? ox : oy;
    int lo = bounds[2 * o], cnt = bounds[2 * o + 1];
    const int* k = kk + (long long)o * ksize;
    int ss = 1 << (RF_PRECISION_BITS - 1);
    if (horizontal) {
        const unsigned char* row = in + ((long long)oy * in_w) * ch + c;
        for (int x = 0; x < cnt; ++x) ss += (int)row[(long long)(x + lo) * ch] * k[x];
    } else {
        const unsigned char* col = in + (long long)ox * ch + c;
        for (int y = 0; y < cnt; ++y) ss += (int)col[(long long)(y + lo) * in_w * ch] * k[y];
    }
    out[t] = clip8(ss);
}

// ---------------------------------------------------------------------------
// homography grid, bilinear sampling, bilinear upsampling, fused composition
// ---------------------------------------------------------------------------
// torch.linspace(-1, 1, n)[i] as the CUDA kernel computes it
__device__ __forceinline__ float lin11(int i, int n) {
    if (n == 1) return -1.f;
    float step = 2.f / (float)(n - 1);
    return (i < n / 2) ? (-1.f + step * (float)i) : (1.f - step * (float)(n - 1 - i));
}

// the grid point of output pixel (r, c) of an h x w homography grid (H: 9 floats), one rounding per operation
__device__ __forceinline__ float2 homography_grid_point(const float* __restrict__ H, int r, int c, int h, int w) {
    float x = lin11(c, w), y = lin11(r, h);
    float px = __fadd_rn(__fadd_rn(__fmul_rn(H[0], x), __fmul_rn(H[1], y)), H[2]);
    float py = __fadd_rn(__fadd_rn(__fmul_rn(H[3], x), __fmul_rn(H[4], y)), H[5]);
    float pz = __fadd_rn(__fadd_rn(__fmul_rn(H[6], x), __fmul_rn(H[7], y)), H[8]);
    return make_float2(__fdiv_rn(px, pz), __fdiv_rn(py, pz));
}

__global__ void warp_grid_kernel(const float* __restrict__ Hm, int N, int h, int w, float* __restrict__ grid) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long hw = (long long)h * w;
    if (t >= N * hw) return;
    int n = (int)(t / hw);
    int rem = (int)(t - n * hw);
    int r = rem / w, c = rem - r * w;
    reinterpret_cast<float2*>(grid)[t] = homography_grid_point(Hm + n * 9, r, c, h, w);
}

__device__ __forceinline__ float unnormalize(float coord, int size, int align_corners) {
    return align_corners ? ((coord + 1.f) / 2.f) * (float)(size - 1) : ((coord + 1.f) * (float)size - 1.f) / 2.f;
}

// torch's CUDA grid sampler moves a source coordinate that is not finite or lies beyond the int range outside the image
// (safe_downgrade_to_int_range), so it samples nothing.  Without this a NaN coordinate would convert to pixel 0 and
// return NaN instead of the 0 F.grid_sample returns.  (|c| = 2^31, which torch keeps, samples nothing either way.)
__device__ __forceinline__ float in_int_range(float c) {
    return fabsf(c) < 2147483648.f ? c : -100.f;
}

struct Strides4 { long long n, c, h, w; };

// F.grid_sample(bilinear, zeros) at one grid point: the top-left tap, the four tap weights and which taps lie inside
struct BilinearTaps {
    int x0, y0;
    float nw, ne, sw, se;
    bool vx0, vx1, vy0, vy1;
};
__device__ __forceinline__ BilinearTaps bilinear_taps(float2 g, int Hin, int Win, int align_corners) {
    BilinearTaps t;
    float ix = in_int_range(unnormalize(g.x, Win, align_corners)), iy = in_int_range(unnormalize(g.y, Hin, align_corners));
    float fx = floorf(ix), fy = floorf(iy);
    t.x0 = (int)fx;
    t.y0 = (int)fy;
    int x1 = t.x0 + 1, y1 = t.y0 + 1;
    t.nw = (fx + 1.f - ix) * (fy + 1.f - iy);
    t.ne = (ix - fx) * (fy + 1.f - iy);
    t.sw = (fx + 1.f - ix) * (iy - fy);
    t.se = (ix - fx) * (iy - fy);
    t.vx0 = t.x0 >= 0 && t.x0 < Win;
    t.vx1 = x1 >= 0 && x1 < Win;
    t.vy0 = t.y0 >= 0 && t.y0 < Hin;
    t.vy1 = y1 >= 0 && y1 < Hin;
    return t;
}
// the inside taps' weighted sum, in nw, ne, sw, se order; load(y, x) reads the input value at an inside tap
template <typename Load>
__device__ __forceinline__ float bilinear_sum(const BilinearTaps& t, Load load) {
    float acc = 0.f;
    if (t.vy0 && t.vx0) acc += load(t.y0, t.x0) * t.nw;
    if (t.vy0 && t.vx1) acc += load(t.y0, t.x0 + 1) * t.ne;
    if (t.vy1 && t.vx0) acc += load(t.y0 + 1, t.x0) * t.sw;
    if (t.vy1 && t.vx1) acc += load(t.y0 + 1, t.x0 + 1) * t.se;
    return acc;
}

__global__ void grid_sample_kernel(const float* __restrict__ in, int N, int C, int Hin, int Win, Strides4 is,
                                   const float* __restrict__ grid, int Hout, int Wout, int align_corners,
                                   float* __restrict__ out, Strides4 os) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long hw = (long long)Hout * Wout;
    if (t >= N * hw) return;
    int n = (int)(t / hw);
    int rem = (int)(t - n * hw);
    int r = rem / Wout, c = rem - r * Wout;
    const BilinearTaps tap = bilinear_taps(__ldg(reinterpret_cast<const float2*>(grid) + t), Hin, Win, align_corners);
    const float* base = in + n * is.n;
    float* ob = out + n * os.n + r * os.h + c * os.w;
    for (int ch = 0; ch < C; ++ch) {
        const float* p = base + ch * is.c;
        ob[ch * os.c] = bilinear_sum(tap, [&](int y, int x) { return __ldg(p + y * is.h + x * is.w); });
    }
}

// train/generate_coarse_aligned_pair.ipynb cell 13 and ToPILImage in one pass: output pixel (r, c) of the h x w homography
// grid of H (device memory), bilinear zero-padded sampling of ToTensor(src) (uint8 HWC / 255, preproc_one), x 255 truncated
// to uint8.  The grid, the fp32 copy of the source and the fp32 sampled image are never stored.
__global__ void __launch_bounds__(256) warp_sample_u8_kernel(const float* __restrict__ H, const unsigned char* __restrict__ src, int Hin,
                                                             int Win, int h, int w, int align_corners, unsigned char* __restrict__ out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)h * w) return;
    int r = (int)(t / w), c = (int)(t - (long long)r * w);
    const BilinearTaps tap = bilinear_taps(homography_grid_point(H, r, c, h, w), Hin, Win, align_corners);
    for (int ch = 0; ch < 3; ++ch) {
        float v = bilinear_sum(tap, [&](int y, int x) { return preproc_one(__ldg(src + ((long long)y * Win + x) * 3 + ch), ch, 0); });
        out[t * 3 + ch] = (unsigned char)__float2uint_rz(__fmul_rn(v, 255.f));
    }
}

// F.affine_grid(theta, (N, C, h, w), align_corners=False) at output pixel (r, c), theta 2 x 3 row-major.  The base coordinate
// is ATen's linspace(-1, 1, n) * (n - 1) / n on the CUDA linspace: the product by n - 1, then the division by the scalar n,
// which ATen's CUDA division performs as a product with the fp32 reciprocal 1 / n; n = 1 gives 0.  theta is applied as one
// FMA chain (x, y, then the constant); torch runs that product as a cuBLAS bmm, so the grid equals torch's to a few ulps
// of its largest term, not bit for bit.
__device__ __forceinline__ float affine_base(int i, int n) {
    if (n <= 1) return 0.f;
    return __fmul_rn(__fmul_rn(lin11(i, n), (float)(n - 1)), __fdiv_rn(1.f, (float)n));
}
__device__ __forceinline__ float2 affine_grid_point(const float* __restrict__ theta, int r, int c, int h, int w) {
    float x = affine_base(c, w), y = affine_base(r, h);
    float px = __fadd_rn(__fmaf_rn(__ldg(theta + 1), y, __fmul_rn(__ldg(theta + 0), x)), __ldg(theta + 2));
    float py = __fadd_rn(__fmaf_rn(__ldg(theta + 4), y, __fmul_rn(__ldg(theta + 3), x)), __ldg(theta + 5));
    return make_float2(px, py);
}

// train/validation.py:80,98-99 in one pass: output pixel (r, c) of the h x w affine grid of theta (device memory), bilinear
// zero-padded sampling (align_corners=False) of ToTensor(src) (uint8 HWC / 255, preproc_one), written as the fp32 NHWC row
// the FeatureExtractor reads.  The grid and the fp32 copy of the source are never stored; a non-finite theta samples zeros.
__global__ void __launch_bounds__(256) affine_sample_u8_kernel(const float* __restrict__ theta, const unsigned char* __restrict__ src,
                                                               int Hin, int Win, int h, int w, float* __restrict__ out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)h * w) return;
    int r = (int)(t / w), c = (int)(t - (long long)r * w);
    const BilinearTaps tap = bilinear_taps(affine_grid_point(theta, r, c, h, w), Hin, Win, 0);
    for (int ch = 0; ch < 3; ++ch)
        out[t * 3 + ch] = bilinear_sum(tap, [&](int y, int x) { return preproc_one(__ldg(src + ((long long)y * Win + x) * 3 + ch), ch, 0); });
}

// F.interpolate(bilinear, align_corners=False) source index / weights
__device__ __forceinline__ void up_coord(int dst, int in_size, int out_size, int& i0, int& i1, float& l0, float& l1) {
    float scale = (float)in_size / (float)out_size;
    float src = scale * ((float)dst + 0.5f) - 0.5f;
    if (src < 0.f) src = 0.f;
    i0 = (int)src;
    i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
    l1 = src - (float)i0;
    l0 = 1.f - l1;
}
// the four taps weighted in ATen's order (rows of the blend first)
__device__ __forceinline__ float up_blend(float v00, float v01, float v10, float v11, float ly0, float ly1, float lx0, float lx1) {
    return ly0 * (lx0 * v00 + lx1 * v01) + ly1 * (lx0 * v10 + lx1 * v11);
}
__device__ __forceinline__ float up_sample(const float* __restrict__ p, int h, int w, int H, int W, int Y, int X) {
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    up_coord(Y, h, H, y0, y1, ly0, ly1);
    up_coord(X, w, W, x0, x1, lx0, lx1);
    return up_blend(__ldg(p + y0 * w + x0), __ldg(p + y0 * w + x1), __ldg(p + y1 * w + x0), __ldg(p + y1 * w + x1), ly0, ly1, lx0, lx1);
}

__global__ void upsample_kernel(const float* __restrict__ in, int NC, int h, int w, int H, int W, float* __restrict__ out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long HW = (long long)H * W;
    if (t >= NC * HW) return;
    int nc = (int)(t / HW);
    int rem = (int)(t - nc * HW);
    int Y = rem / W, X = rem - Y * W;
    out[t] = up_sample(in + (long long)nc * h * w, h, w, H, W, Y, X);
}

// train/validation.py:93-107 and alignmentError (:33-53) at the annotated keypoints only.  Per keypoint (xa, ya, xb, yb):
// torch's index rule on (yb, xb) in the H x W target (a negative index wraps once; anything else records the pair in *err);
// F.upsample_bilinear (align_corners=True) of flowDown8 at that pixel with ATen's CUDA arithmetic (fp32 scale, (int) floor,
// the h1p / w1p edge step, the lambda order of up_blend); + the grid of validation.py:93-95, a CPU torch.linspace, which
// lin11 reproduces (ATen's AVX2 / AVX-512 CPU kernel contracts both branches into one FMA, as nvcc does here: the scalar
// "default" build, which rounds twice, differs by an ulp in places); clamped to [-1, 1] with NaN kept; the
// F.grid_sample (bilinear, zeros, align_corners=False) of the H x W affine grid of theta at that point, its four taps
// recomputed; estim = (flow + 1) * 0.5 * (size - 1) in fp32 (wA, hA: the resized source); the distance to (xa, ya) in fp64;
// counts[t] += (dist < thresholds[t]) and counts[T] += 1 over the block, one atomic per counter.
#define RF_VAL_MAX_THRESHOLDS 16
struct ValThresholds { double t[RF_VAL_MAX_THRESHOLDS]; int n; };

__device__ __forceinline__ float clamp11_nan(float v) { return isnan(v) ? v : fminf(fmaxf(v, -1.f), 1.f); }

__global__ void __launch_bounds__(256) val_keypoints_kernel(const float* __restrict__ flow8, int h8, int w8, const float* __restrict__ theta,
                                                            int H, int W, int wA, int hA, const int* __restrict__ kpts,
                                                            const int* __restrict__ count, int capacity, int pair,
                                                            const __grid_constant__ ValThresholds th, unsigned long long* __restrict__ counts,
                                                            int* __restrict__ err, double* __restrict__ dist_out, float* __restrict__ flow_out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(__ldg(count), capacity);
    bool live = j < n;
    double dist = 0.0;
    if (live) {
        const int xa = __ldg(kpts + 4 * j), ya = __ldg(kpts + 4 * j + 1);
        int xb = __ldg(kpts + 4 * j + 2), yb = __ldg(kpts + 4 * j + 3);
        if (yb < 0 && yb >= -H) yb += H;
        if (xb < 0 && xb >= -W) xb += W;
        if (yb < 0 || yb >= H || xb < 0 || xb >= W) {
            atomicMin(err, pair);
            live = false;
            if (dist_out) dist_out[j] = __longlong_as_double(0x7ff8000000000000ll);
        } else {
            const float rh = H > 1 ? __fdiv_rn((float)(h8 - 1), (float)(H - 1)) : 0.f;
            const float rw = W > 1 ? __fdiv_rn((float)(w8 - 1), (float)(W - 1)) : 0.f;
            const float h1r = __fmul_rn(rh, (float)yb), w1r = __fmul_rn(rw, (float)xb);
            const int h1 = (int)h1r, w1 = (int)w1r;
            const int h1p = h1 < h8 - 1 ? 1 : 0, w1p = w1 < w8 - 1 ? 1 : 0;
            const float h1l = h1r - (float)h1, w1l = w1r - (float)w1;
            const float h0l = 1.f - h1l, w0l = 1.f - w1l;
            const float* p0 = flow8 + (long long)h1 * w8 + w1;
            const float* p1 = p0 + (long long)h8 * w8;
            const long long dy = (long long)h1p * w8;
            float fx = up_blend(__ldg(p0), __ldg(p0 + w1p), __ldg(p0 + dy), __ldg(p0 + dy + w1p), h0l, h1l, w0l, w1l);
            float fy = up_blend(__ldg(p1), __ldg(p1 + w1p), __ldg(p1 + dy), __ldg(p1 + dy + w1p), h0l, h1l, w0l, w1l);
            fx = clamp11_nan(__fadd_rn(fx, lin11(xb, W)));
            fy = clamp11_nan(__fadd_rn(fy, lin11(yb, H)));
            const BilinearTaps tap = bilinear_taps(make_float2(fx, fy), H, W, 0);
            const float ox = bilinear_sum(tap, [&](int y, int x) { return affine_grid_point(theta, y, x, H, W).x; });
            const float oy = bilinear_sum(tap, [&](int y, int x) { return affine_grid_point(theta, y, x, H, W).y; });
            if (flow_out) reinterpret_cast<float4*>(flow_out)[j] = make_float4(fx, fy, ox, oy);
            const float ex = __fmul_rn(__fmul_rn(__fadd_rn(ox, 1.f), 0.5f), (float)(wA - 1));
            const float ey = __fmul_rn(__fmul_rn(__fadd_rn(oy, 1.f), 0.5f), (float)(hA - 1));
            const double ddx = __dsub_rn((double)ex, (double)xa), ddy = __dsub_rn((double)ey, (double)ya);
            dist = __dsqrt_rn(__dadd_rn(__dmul_rn(ddx, ddx), __dmul_rn(ddy, ddy)));
            if (dist_out) dist_out[j] = dist;
        }
    }
    for (int t = 0; t < th.n; ++t) {
        const int c = __syncthreads_count(live && dist < th.t[t]);
        if (threadIdx.x == 0 && c) atomicAdd(counts + t, (unsigned long long)c);
    }
    const int c = __syncthreads_count(live);
    if (threadIdx.x == 0 && c) atomicAdd(counts + th.n, (unsigned long long)c);
}

// evaluation/evalHpatch/evaluation.py:37-51 (and evalCorr :50-55) in one pass over the full-res grid.  The coarse grid
// may have its own size (Hc, Wc) != (H, W): evaluation/evalKITTI/evaluation.py:296-299 samples the flow of the resized
// image at the original image's positions, and evalKITTI/getResults.py:104-113 composes two levels that way.
__global__ void compose_fine_kernel(const float* __restrict__ flow8, const float* __restrict__ m12, const float* __restrict__ m21,
                                    int h8, int w8, const float* __restrict__ coarse, int Hc, int Wc, int H, int W, int clamp, int align_corners,
                                    float* __restrict__ flow12, float* __restrict__ match, float* __restrict__ flowUp_out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)H * W) return;
    int Y = (int)(t / W), X = (int)(t - (long long)Y * W);
    float fx = up_sample(flow8, h8, w8, H, W, Y, X) + lin11(X, W);
    float fy = up_sample(flow8 + h8 * w8, h8, w8, H, W, Y, X) + lin11(Y, H);
    if (clamp) {
        fx = fminf(fmaxf(fx, -1.f), 1.f);
        fy = fminf(fmaxf(fy, -1.f), 1.f);
    }
    if (flowUp_out) reinterpret_cast<float2*>(flowUp_out)[t] = make_float2(fx, fy);
    const float2* cg = reinterpret_cast<const float2*>(coarse);
    float ox = 0.f, oy = 0.f, mm = 0.f;
    {   // grid_sample(coarse, flowUp): bilinear, zero padding, in the coarse grid's own pixel coordinates
        float ix = unnormalize(fx, Wc, align_corners), iy = unnormalize(fy, Hc, align_corners);
        float flx = floorf(ix), fly = floorf(iy);
        int x0 = (int)flx, y0 = (int)fly, x1 = x0 + 1, y1 = y0 + 1;
        float nw = (flx + 1.f - ix) * (fly + 1.f - iy), ne = (ix - flx) * (fly + 1.f - iy);
        float sw = (flx + 1.f - ix) * (iy - fly), se = (ix - flx) * (iy - fly);
        bool vx0 = x0 >= 0 && x0 < Wc, vx1 = x1 >= 0 && x1 < Wc, vy0 = y0 >= 0 && y0 < Hc, vy1 = y1 >= 0 && y1 < Hc;
        if (vy0 && vx0) { float2 v = __ldg(cg + (long long)y0 * Wc + x0); ox += v.x * nw; oy += v.y * nw; }
        if (vy0 && vx1) { float2 v = __ldg(cg + (long long)y0 * Wc + x1); ox += v.x * ne; oy += v.y * ne; }
        if (vy1 && vx0) { float2 v = __ldg(cg + (long long)y1 * Wc + x0); ox += v.x * sw; oy += v.y * sw; }
        if (vy1 && vx1) { float2 v = __ldg(cg + (long long)y1 * Wc + x1); ox += v.x * se; oy += v.y * se; }
    }
    if (m21) {   // grid_sample(interpolate(match21, (H, W)), flowUp): the sampled map lives on the OUTPUT grid
        float ix = unnormalize(fx, W, align_corners), iy = unnormalize(fy, H, align_corners);
        float flx = floorf(ix), fly = floorf(iy);
        int x0 = (int)flx, y0 = (int)fly, x1 = x0 + 1, y1 = y0 + 1;
        float nw = (flx + 1.f - ix) * (fly + 1.f - iy), ne = (ix - flx) * (fly + 1.f - iy);
        float sw = (flx + 1.f - ix) * (iy - fly), se = (ix - flx) * (iy - fly);
        bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
        if (vy0 && vx0) mm += up_sample(m21, h8, w8, H, W, y0, x0) * nw;
        if (vy0 && vx1) mm += up_sample(m21, h8, w8, H, W, y0, x1) * ne;
        if (vy1 && vx0) mm += up_sample(m21, h8, w8, H, W, y1, x0) * sw;
        if (vy1 && vx1) mm += up_sample(m21, h8, w8, H, W, y1, x1) * se;
    }
    reinterpret_cast<float2*>(flow12)[t] = make_float2(ox, oy);
    if (match) {
        float m = up_sample(m12, h8, w8, H, W, Y, X);
        if (m21) m *= mm;
        float inside = ((ox >= -1.f && ox <= 1.f) ? 1.f : 0.f) * ((oy >= -1.f && oy <= 1.f) ? 1.f : 0.f);
        match[t] = m * inside;
    }
}

// ---------------------------------------------------------------------------
// remove_small_cc (evaluation/evalKITTI/evaluation.py:85-100, evalKITTI/getResults.py:66-83): zero the matchability of
// every 8-connected component of (match > match_th) whose area fraction is <= cc_th.  skimage.measure.label's default
// connectivity for a 2-D array is 2 (8 neighbours).  Label-equivalence union-find (one pass over the four "backward"
// neighbours, atomicMin roots), then flatten, count, filter.
// ---------------------------------------------------------------------------
__device__ __forceinline__ int cc_find(const int* L, int i) {
    int p = L[i];
    while (p != i) { i = p; p = L[i]; }
    return i;
}
__device__ __forceinline__ void cc_union(int* L, int a, int b) {
    bool done = false;
    while (!done) {
        a = cc_find(L, a);
        b = cc_find(L, b);
        if (a < b) { int old = atomicMin(&L[b], a); done = (old == b); b = old; }
        else if (b < a) { int old = atomicMin(&L[a], b); done = (old == a); a = old; }
        else done = true;
    }
}
__global__ void cc_init_kernel(const float* __restrict__ match, float th, int n, int* __restrict__ L, int* __restrict__ cnt) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    L[i] = (match[i] > th) ? i : -1;
    cnt[i] = 0;
}
__global__ void cc_merge_kernel(int* __restrict__ L, int H, int W) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W || L[i] < 0) return;
    const int y = i / W, x = i - y * W;
    if (x > 0 && L[i - 1] >= 0) cc_union(L, i, i - 1);
    if (y > 0) {
        if (L[i - W] >= 0) cc_union(L, i, i - W);
        if (x > 0 && L[i - W - 1] >= 0) cc_union(L, i, i - W - 1);
        if (x + 1 < W && L[i - W + 1] >= 0) cc_union(L, i, i - W + 1);
    }
}
__global__ void cc_flatten_count_kernel(int* __restrict__ L, int n, int* __restrict__ cnt) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || L[i] < 0) return;
    const int r = cc_find(L, i);
    atomicAdd(&cnt[r], 1);
    // L[i] is rewritten in the next kernel (roots must stay intact while other threads still walk to them)
}
__global__ void cc_filter_kernel(float* __restrict__ match, const int* __restrict__ L, const int* __restrict__ cnt, int n, double cc_th) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || L[i] < 0) return;
    const int r = cc_find(L, i);
    if ((double)cnt[r] / (double)n <= cc_th) match[i] = 0.f;         // np.mean(all_labels == i) <= cc_th
}

// ---------------------------------------------------------------------------
// interpolate_flow_match (evaluation/evalKITTI/getResults.py:87-93): every unmatched pixel takes the flow of its nearest
// matched pixel (exact Euclidean distance; scipy.ndimage.distance_transform_edt(return_indices=True) in the reference).
// Exact two-pass feature transform in integer arithmetic: (1) per column, the nearest matched row above / below;
// (2) per row, the lower envelope of the parabolas (x - x')^2 + dy(x')^2 (Felzenszwalb & Huttenlocher), then the gather.
// Between equidistant matched pixels the choice is: smaller |dy| column-wise first (ties -> the row above), then the
// envelope's left-most parabola; scipy resolves such ties in its own order, so outputs can differ there (and only there).
// ---------------------------------------------------------------------------
__global__ void edt_cols_kernel(const unsigned char* __restrict__ matched, int H, int W, int* __restrict__ gy) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    int last = -1;
    for (int y = 0; y < H; ++y) {
        if (matched[(long long)y * W + x]) last = y;
        gy[(long long)y * W + x] = last;
    }
    last = -1;
    for (int y = H - 1; y >= 0; --y) {
        if (matched[(long long)y * W + x]) last = y;
        const int a = gy[(long long)y * W + x];
        int pick = a;
        if (a < 0) pick = last;
        else if (last >= 0 && (last - y) < (y - a)) pick = last;
        gy[(long long)y * W + x] = pick;
    }
}
__global__ void edt_rows_fill_kernel(const int* __restrict__ gy, int H, int W, int* __restrict__ v, double* __restrict__ z,
                                     const float2* __restrict__ flow, float2* __restrict__ out, int* __restrict__ idx_out) {
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= H) return;
    const int* g = gy + (long long)y * W;
    int* vv = v + (long long)y * W;
    double* zz = z + (long long)y * (W + 1);
    int k = -1;
    for (int q = 0; q < W; ++q) {
        if (g[q] < 0) continue;
        const long long dq = (long long)(y - g[q]) * (y - g[q]);
        double sx = -1e300;
        while (k >= 0) {
            const int p = vv[k];
            const long long dp = (long long)(y - g[p]) * (y - g[p]);
            sx = (double)((dq + (long long)q * q) - (dp + (long long)p * p)) / (double)(2 * (q - p));
            if (sx <= zz[k]) --k; else break;
        }
        if (k < 0) sx = -1e300;
        ++k;
        vv[k] = q;
        zz[k] = sx;
    }
    if (k < 0) {                                   // no matched pixel at all: leave the row as it is
        for (int x = 0; x < W; ++x) { out[(long long)y * W + x] = flow[(long long)y * W + x]; if (idx_out) { idx_out[2 * ((long long)y * W + x)] = y; idx_out[2 * ((long long)y * W + x) + 1] = x; } }
        return;
    }
    const int kmax = k;
    k = 0;
    for (int x = 0; x < W; ++x) {
        while (k < kmax && zz[k + 1] < (double)x) ++k;
        const int xs = vv[k], ys = g[xs];
        out[(long long)y * W + x] = flow[(long long)ys * W + xs];
        if (idx_out) { idx_out[2 * ((long long)y * W + x)] = ys; idx_out[2 * ((long long)y * W + x) + 1] = xs; }
    }
}

}  // namespace rf

using namespace rf;

static inline unsigned blocks_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// CorrNeigh(x, y) into `out` (and CorrNeigh(y, x) into `out2`, nullable): the register-accumulating kernel for k = 7, the
// one-reduction-per-tap kernel for other odd k
static int launch_corr_neigh(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, int round_out, float* out,
                             float* out2, void* stream) {
    const long long P = (long long)N * h * w;
    if (P == 0) return 0;
    if (k == 7) corr_neigh7_kernel<<<blocks_for(P * 32, 256), 256, 0, as_stream(stream)>>>(x, y, N, h, w, C, ldo, round_out, out, out2);
    else corr_neigh_kernel<<<blocks_for(P * 32, 256), 256, 0, as_stream(stream)>>>(x, y, N, h, w, C, k, ldo, round_out, out, out2);
    RF_LAUNCHED();
    return 0;
}

// ---- the layer ops of rf_run_layers, one launcher per op over the activation format ----
// Vec16 width of a format: the channel count must be a multiple of it
static int vec_width(ActFormat f) { return f == ACT_F16 || f == ACT_SPLIT ? 8 : 4; }

// launch(T()) with the Vec16 type of the format: float (fp32, TF32), __half (fp16) or SplitH (split)
template <typename Launch>
static void for_format(ActFormat f, Launch&& launch) {
    if (f == ACT_F16) launch(__half());
    else if (f == ACT_SPLIT) launch(SplitH());
    else launch(float());
}

// One thread per (output pixel, 16-byte vector).  Split planes are the whole input / output tensors apart; the other formats
// ignore pin / pout.
int rf_maxpool(ActFormat f, const void* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, void* y, void* stream) {
    const int vn = vec_width(f);
    RF_REQUIRE((C % vn) == 0 && k >= 1 && stride >= 1, "rf_maxpool: C must be a multiple of 4 (fp32) or 8 (fp16, split)");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, k, stride, pad) == 0, "rf_maxpool: bad image set");
    const unsigned blocks = blocks_for(set.out_pix[nimg] * (C / vn), 256);
    for_format(f, [&](auto t) {
        typedef typename Vec16<decltype(t)>::elem E;
        maxpool_kernel<decltype(t)><<<blocks, 256, 0, as_stream(stream)>>>(set, static_cast<const E*>(x), static_cast<E*>(y), C, k, stride, pad,
                                                                           set.in_pix[nimg] * C, set.out_pix[nimg] * C);
    });
    RF_LAUNCHED();
    return 0;
}

int rf_blur(ActFormat f, const void* x, int nimg, const int* hw_host, int C, int stride, void* y, void* stream) {
    const int vn = vec_width(f);
    RF_REQUIRE((C % vn) == 0 && stride >= 1, "rf_blur: C must be a multiple of 4 (fp32) or 8 (fp16, split)");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 3, stride, 1) == 0, "rf_blur: bad image set");
    for (int i = 0; i < nimg; ++i) RF_REQUIRE(set.H[i] >= 2 && set.W[i] >= 2, "rf_blur: reflect padding needs H, W >= 2");
    const unsigned blocks = blocks_for(set.out_pix[nimg] * (C / vn), 256);
    for_format(f, [&](auto t) {
        typedef typename Vec16<decltype(t)>::elem E;
        blur_kernel<decltype(t)><<<blocks, 256, 0, as_stream(stream)>>>(set, static_cast<const E*>(x), static_cast<E*>(y), C, stride, f == ACT_TF32,
                                                                        set.in_pix[nimg] * C, set.out_pix[nimg] * C);
    });
    RF_LAUNCHED();
    return 0;
}

// output size of maxpool(2,1) + blur(stride 2): ((H-1) + 2 - 3)/2 + 1 = make_imgset with k = 4, stride 2, pad 1
int rf_poolblur(ActFormat f, const void* x, int nimg, const int* hw_host, int C, void* y, void* stream) {
    const int vn = vec_width(f);
    RF_REQUIRE((C % vn) == 0, "rf_poolblur: C must be a multiple of 4 (fp32) or 8 (fp16, split)");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 4, 2, 1) == 0, "rf_poolblur: bad image set");
    for (int i = 0; i < nimg; ++i) RF_REQUIRE(set.H[i] >= 3 && set.W[i] >= 3, "rf_poolblur: needs H, W >= 3");
    const unsigned blocks = blocks_for(set.out_pix[nimg] * (C / vn), 256);
    for_format(f, [&](auto t) {
        typedef typename Vec16<decltype(t)>::elem E;
        poolblur_kernel<decltype(t)><<<blocks, 256, 0, as_stream(stream)>>>(set, static_cast<const E*>(x), static_cast<E*>(y), C, f == ACT_TF32,
                                                                            set.in_pix[nimg] * C, set.out_pix[nimg] * C);
    });
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_maxpool2d_nhwc(const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, float* y, void* stream) {
    return rf_maxpool(ACT_F32, x, nimg, hw_host, C, k, stride, pad, y, stream);
}

extern "C" int rf_blur_downsample_nhwc(const float* x, int nimg, const int* hw_host, int C, int stride, float* y, void* stream) {
    return rf_blur(ACT_F32, x, nimg, hw_host, C, stride, y, stream);
}

// Stem-specialised im2col: one CTA = one output row segment of TPX pixels.  The K input rows it needs are staged in
// shared memory with coalesced loads, then the (r, s, c)-ordered patches are written as contiguous rows of 16-byte vectors.
template <int K, int C, int KPAD, int STRIDE, int PAD, int TPX, typename OutT = float>
__global__ void __launch_bounds__(256)
im2col_smem_kernel(const __grid_constant__ ImgSet set, const float* __restrict__ x, typename Vec16<OutT>::elem* __restrict__ y, int round_out,
                   long long plane = 0) {
    constexpr int INW = ((TPX - 1) * STRIDE + K) * C;          // floats of one staged input row
    constexpr int VN = Vec16<OutT>::N, QV = KPAD / VN;
    __shared__ float sIn[K][INW + 1];
    const int im = blockIdx.z, oy = blockIdx.y, ox0 = blockIdx.x * TPX;
    const int Wo = set.Wo[im];
    if (oy >= set.Ho[im] || ox0 >= Wo) return;
    const int H = set.H[im], WC = set.W[im] * C;
    const float* src = x + set.in_pix[im] * C;
    const int col0 = (ox0 * STRIDE - PAD) * C;
    // all global loads first (independent: one DRAM latency for the whole window), then the shared-memory stores
    constexpr int NLD = (K * INW + 255) / 256;
    float stage[NLD];
#pragma unroll
    for (int i = 0; i < NLD; ++i) {
        const int idx = threadIdx.x + i * 256;
        const int r = idx / INW, j = idx - r * INW;
        const int iy = oy * STRIDE - PAD + r, col = col0 + j;
        stage[i] = (idx < K * INW && iy >= 0 && iy < H && col >= 0 && col < WC) ? __ldg(src + (long long)iy * WC + col) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < NLD; ++i) {
        const int idx = threadIdx.x + i * 256;
        const int r = idx / INW, j = idx - r * INW;
        if (idx < K * INW) sIn[r][j] = round_out ? round_tf32(stage[i]) : stage[i];
    }
    __syncthreads();
    const int npx = min(TPX, Wo - ox0);
    typename Vec16<OutT>::elem* dst = y + (set.out_pix[im] + (long long)oy * Wo + ox0) * KPAD;
    for (int f = threadIdx.x; f < npx * QV; f += 256) {
        const int px = f / QV, e0 = (f - px * QV) * VN;
        float v[VN];
#pragma unroll
        for (int j = 0; j < VN; ++j) {
            const int e = e0 + j;
            v[j] = (e < K * K * C) ? sIn[e / (K * C)][px * STRIDE * C + e % (K * C)] : 0.f;
        }
        Vec16<OutT>::store(dst + (long long)f * VN, plane, v, 0);
    }
}

// fp32 / TF32: any shape (the two stems on the shared-memory kernel).  fp16 rows only for the ResNet-50 stem (7x7/2, Kpad 192)
// and the FeatureExtractor stem (3x3/1, Kpad 64); split rows only for the FeatureExtractor stem.
int rf_im2col(ActFormat f, const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad, int Kpad, void* y, void* stream) {
    const bool f32 = f == ACT_F32 || f == ACT_TF32;
    const bool resnet = k == 7 && C == 3 && stride == 2 && pad == 3 && Kpad == (f32 ? 160 : 192);
    const bool fe = k == 3 && C == 3 && stride == 1 && pad == 1 && Kpad == (f32 ? 32 : 64);
    RF_REQUIRE(f != ACT_F16 || resnet || fe, "rf_im2col (fp16): only the ResNet-50 stem (7x7/2, Kpad 192) and the FeatureExtractor stem (3x3/1, Kpad 64)");
    RF_REQUIRE(f != ACT_SPLIT || fe, "rf_im2col (split): only the FeatureExtractor stem (3x3/1, Kpad 64)");
    RF_REQUIRE(Kpad >= k * k * C && C >= 1, "rf_im2col: Kpad too small");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, k, stride, pad) == 0, "rf_im2col: bad image set");
    RF_REQUIRE((Kpad & 3) == 0, "rf_im2col: Kpad must be a multiple of 4");
    long long maxq = 0;
    int maxHo = 0, maxWo = 0;
    for (int i = 0; i < nimg; ++i) {
        const long long q = (long long)set.Ho[i] * set.Wo[i] * (Kpad / 4);
        RF_REQUIRE(!f32 || q < (1ll << 31), "rf_im2col: image too large for 32-bit indexing");
        maxq = q > maxq ? q : maxq;
        maxHo = set.Ho[i] > maxHo ? set.Ho[i] : maxHo;
        maxWo = set.Wo[i] > maxWo ? set.Wo[i] : maxWo;
    }
    const int round_out = f == ACT_TF32;
    const dim3 grid_resnet((maxWo + 63) / 64, maxHo, nimg), grid_fe((maxWo + 127) / 128, maxHo, nimg);
    cudaStream_t st = as_stream(stream);
    float* y32 = static_cast<float*>(y);
    __half* y16 = static_cast<__half*>(y);
    if (f == ACT_SPLIT) im2col_smem_kernel<3, 3, 64, 1, 1, 128, SplitH><<<grid_fe, 256, 0, st>>>(set, x, y16, 0, set.out_pix[nimg] * 64);
    else if (f == ACT_F16 && resnet) im2col_smem_kernel<7, 3, 192, 2, 3, 64, __half><<<grid_resnet, 256, 0, st>>>(set, x, y16, 0);
    else if (f == ACT_F16) im2col_smem_kernel<3, 3, 64, 1, 1, 128, __half><<<grid_fe, 256, 0, st>>>(set, x, y16, 0);
    else if (resnet) im2col_smem_kernel<7, 3, 160, 2, 3, 64><<<grid_resnet, 256, 0, st>>>(set, x, y32, round_out);
    else if (fe) im2col_smem_kernel<3, 3, 32, 1, 1, 128><<<grid_fe, 256, 0, st>>>(set, x, y32, round_out);
    else {
        const dim3 grid(blocks_for(maxq, 256), nimg);
        if (k == 7 && C == 3 && Kpad == 160) im2col_kernel<7, 3, 160><<<grid, 256, 0, st>>>(set, x, y32, C, k, stride, pad, Kpad, round_out);
        else if (k == 3 && C == 3 && Kpad == 32) im2col_kernel<3, 3, 32><<<grid, 256, 0, st>>>(set, x, y32, C, k, stride, pad, Kpad, round_out);
        else im2col_kernel<0, 0, 0><<<grid, 256, 0, st>>>(set, x, y32, C, k, stride, pad, Kpad, round_out);
    }
    RF_LAUNCHED();
    return 0;
}

// P rows of C channels (C a multiple of the format's Vec16 width; split planes P * C elements apart) -> fp32 rows / split planes
template <typename T>
static int launch_l2norm(const void* x, long long P, int C, const uint8_t* mask, float* y, void* y_hi, void* y_lo, void* stream) {
    if (P == 0) return 0;
    l2norm_kernel<T><<<blocks_for(P * 32, 256), 256, 0, as_stream(stream)>>>(static_cast<const typename Vec16<T>::elem*>(x), P * C, P, C, mask, y,
                                                                              static_cast<__half*>(y_hi), static_cast<__half*>(y_lo));
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_l2norm_f16_nhwc(const void* x_f16, long long P, int C, const uint8_t* mask, float* y, void* stream) {
    RF_REQUIRE((C % 8) == 0 && P >= 0, "rf_l2norm_f16_nhwc: C must be a multiple of 8");
    RF_REQUIRE(((uintptr_t)x_f16 % 16) == 0 && ((uintptr_t)y % 16) == 0, "rf_l2norm_f16_nhwc: pointers must be 16-byte aligned");
    return launch_l2norm<__half>(x_f16, P, C, mask, y, nullptr, nullptr, stream);
}

// segNet's deep-stem conv1 (segNet/segModel.py:64,108): 3x3 / stride 2 / pad 1 on the 3-channel fp32 image + folded BN + ReLU ->
// split [2][sum HoWo][64].  27 multiply-adds per output: exact fp32 FMA, one thread per (output pixel, 8 channels); the weights
// w [27][64] ((r, s, c) rows) are staged in shared memory.  No patch matrix goes to HBM.
__global__ void __launch_bounds__(256) stem3_split_kernel(const __grid_constant__ ImgSet set, const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, __half* __restrict__ y, long long plane) {
    __shared__ float sw[27 * 64];
    for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) sw[i] = __ldg(w + i);
    __syncthreads();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= set.out_pix[set.n] * 8) return;
    const long long pix = t >> 3;
    const int c0 = (int)(t & 7) * 8;
    const int im = find_img(set, pix);
    const int Wo = set.Wo[im], H = set.H[im], W = set.W[im];
    const int rem = (int)(pix - set.out_pix[im]), oy = rem / Wo, ox = rem - oy * Wo;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = bias ? __ldg(bias + c0 + e) : 0.f;
    const float* src = x + set.in_pix[im] * 3;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int iy = 2 * oy - 1 + r;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            const int ix = 2 * ox - 1 + s;
            if (ix < 0 || ix >= W) continue;
            const float* p = src + ((long long)iy * W + ix) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float v = __ldg(p + c);
                const float* wr = sw + ((r * 3 + s) * 3 + c) * 64 + c0;
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = fmaf(v, wr[e], acc[e]);
            }
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = fmaxf(acc[e], 0.f);
    split_store8(y + pix * 64 + c0, plane, acc);
}

int rf_stem3(const float* x, int nimg, const int* hw_host, const float* w, const float* bias, void* y, void* stream) {
    RF_REQUIRE(x != nullptr && w != nullptr && y != nullptr && ((uintptr_t)y % 16) == 0, "rf_stem3 (engine 4): null or misaligned pointer");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 3, 2, 1) == 0, "rf_stem3: bad image set");
    const long long total = set.out_pix[nimg] * 8;
    stem3_split_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(set, x, w, bias, static_cast<__half*>(y), set.out_pix[nimg] * 64);
    RF_LAUNCHED();
    return 0;
}

// ---- segNet decoder and vote (segNet/segModel.py:218-264, segNet/segEval.py:23-43) on split tensors ----
#define RF_SEG_MAX_BINS 8
struct PoolBins {
    int nbins, bins[RF_SEG_MAX_BINS];
    long long work_start[RF_SEG_MAX_BINS + 1];   // prefix sums of nimg * b * b * C / 8 over the bin counts
    __half* y[RF_SEG_MAX_BINS];
};

// nn.AdaptiveAvgPool2d(b): one thread per (bin count, image, output cell, 8 channels); sums in fp32 in row-major order, then / area
__global__ void adaptive_avgpool_split_kernel(const __grid_constant__ ImgSet set, const __half* __restrict__ x, long long in_plane, int C,
                                              const __grid_constant__ PoolBins pb) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= pb.work_start[pb.nbins]) return;
    int j = 0;
#pragma unroll
    for (int q = 1; q < RF_SEG_MAX_BINS; ++q) j += (q < pb.nbins && t >= pb.work_start[q]) ? 1 : 0;
    const int b = pb.bins[j], C8 = C / 8;
    const long long r = t - pb.work_start[j];
    const int c0 = (int)(r % C8) * 8;
    const long long cell = r / C8;                 // image * b * b + oy * b + ox
    const int im = (int)(cell / (b * b)), oyx = (int)(cell - (long long)im * b * b), oy = oyx / b, ox = oyx - oy * b;
    const int H = set.H[im], W = set.W[im];
    const int y0 = (oy * H) / b, y1 = ((oy + 1) * H + b - 1) / b, x0 = (ox * W) / b, x1 = ((ox + 1) * W + b - 1) / b;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const __half* src = x + set.in_pix[im] * C + c0;
    for (int yy = y0; yy < y1; ++yy)
        for (int xx = x0; xx < x1; ++xx) {
            float v[8];
            split_load8(src + ((long long)yy * W + xx) * C, in_plane, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += v[e];
        }
    const float area = (float)((y1 - y0) * (x1 - x0));
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] /= area;
    split_store8(pb.y[j] + cell * C + c0, (long long)set.n * b * b * C, acc);
}

extern "C" int rf_adaptive_avgpool_split(const void* x, int nimg, const int* hw_host, int C, const int* bins_host, int nbins, void* const* y_host,
                                         void* stream) {
    RF_REQUIRE(x != nullptr && bins_host != nullptr && y_host != nullptr && (C % 8) == 0 && C >= 8 && nbins >= 1 && nbins <= RF_SEG_MAX_BINS,
               "rf_adaptive_avgpool_split: bad arguments (C % 8 == 0, 1 <= nbins <= 8)");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 1, 1, 0) == 0, "rf_adaptive_avgpool_split: bad image set");
    PoolBins pb;
    memset(&pb, 0, sizeof(pb));
    pb.nbins = nbins;
    for (int j = 0; j < nbins; ++j) {
        RF_REQUIRE(bins_host[j] >= 1 && bins_host[j] <= 64 && y_host[j] != nullptr && ((uintptr_t)y_host[j] % 16) == 0,
                   "rf_adaptive_avgpool_split: bin counts 1..64, 16-byte aligned outputs");
        pb.bins[j] = bins_host[j];
        pb.y[j] = static_cast<__half*>(y_host[j]);
        pb.work_start[j + 1] = pb.work_start[j] + (long long)nimg * bins_host[j] * bins_host[j] * (C / 8);
    }
    for (int j = nbins; j < RF_SEG_MAX_BINS; ++j) pb.work_start[j + 1] = pb.work_start[nbins];
    const long long total = pb.work_start[nbins];
    adaptive_avgpool_split_kernel<<<blocks_for(total, 128), 128, 0, as_stream(stream)>>>(set, static_cast<const __half*>(x), set.in_pix[nimg] * C, C, pb);
    RF_LAUNCHED();
    return 0;
}

struct PpmBranches {
    int nbins, bins[RF_SEG_MAX_BINS];
    const __half* src[RF_SEG_MAX_BINS];
};

// [conv5 | up(branch 0) | ... ]: one thread per (pixel, 8 output channels)
__global__ void ppm_concat_split_kernel(const __grid_constant__ ImgSet set, const __half* __restrict__ conv5, int C5, const __grid_constant__ PpmBranches br,
                                       int Cb, __half* __restrict__ y, int Cy) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int Cy8 = Cy / 8;
    const long long P = set.in_pix[set.n];
    if (t >= P * Cy8) return;
    const long long pix = t / Cy8;
    const int c0 = (int)(t - pix * Cy8) * 8;
    __half* dst = y + pix * Cy + c0;
    const long long out_plane = P * Cy;
    if (c0 < C5) {                                  // conv5: the hi / lo halves are copied as they are
        const __half* s = conv5 + pix * C5 + c0;
        *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(s));
        *reinterpret_cast<uint4*>(dst + out_plane) = __ldg(reinterpret_cast<const uint4*>(s + P * C5));
        return;
    }
    const int j = (c0 - C5) / Cb, cb = c0 - C5 - j * Cb, b = br.bins[j];
    int im = 0;
#pragma unroll
    for (int q = 1; q < RF_MAX_IMGS; ++q) im += (q < set.n && pix >= set.in_pix[q]) ? 1 : 0;
    const int H = set.H[im], W = set.W[im];
    const int rem = (int)(pix - set.in_pix[im]), Y = rem / W, X = rem - Y * W;
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    up_coord(Y, b, H, y0, y1, ly0, ly1);
    up_coord(X, b, W, x0, x1, lx0, lx1);
    const __half* s = br.src[j] + ((long long)im * b * b) * Cb + cb;
    const long long in_plane = (long long)set.n * b * b * Cb;
    float v00[8], v01[8], v10[8], v11[8], o[8];
    split_load8(s + (long long)(y0 * b + x0) * Cb, in_plane, v00);
    split_load8(s + (long long)(y0 * b + x1) * Cb, in_plane, v01);
    split_load8(s + (long long)(y1 * b + x0) * Cb, in_plane, v10);
    split_load8(s + (long long)(y1 * b + x1) * Cb, in_plane, v11);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = up_blend(v00[e], v01[e], v10[e], v11[e], ly0, ly1, lx0, lx1);
    split_store8(dst, out_plane, o);
}

extern "C" int rf_ppm_concat_split(const void* conv5, int nimg, const int* hw_host, int C5, void* const* branches_host, const int* bins_host, int nbins,
                                   int Cb, void* y, void* stream) {
    RF_REQUIRE(conv5 != nullptr && y != nullptr && branches_host != nullptr && bins_host != nullptr && nbins >= 1 && nbins <= RF_SEG_MAX_BINS &&
               (C5 % 8) == 0 && (Cb % 8) == 0 && C5 >= 8 && Cb >= 8, "rf_ppm_concat_split: bad arguments (C5 % 8 == Cb % 8 == 0, 1 <= nbins <= 8)");
    RF_REQUIRE(((uintptr_t)conv5 % 16) == 0 && ((uintptr_t)y % 16) == 0, "rf_ppm_concat_split: pointers must be 16-byte aligned");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 1, 1, 0) == 0, "rf_ppm_concat_split: bad image set");
    PpmBranches br;
    memset(&br, 0, sizeof(br));
    br.nbins = nbins;
    for (int j = 0; j < nbins; ++j) {
        RF_REQUIRE(bins_host[j] >= 1 && branches_host[j] != nullptr && ((uintptr_t)branches_host[j] % 16) == 0,
                   "rf_ppm_concat_split: bin counts >= 1, 16-byte aligned branches");
        br.bins[j] = bins_host[j];
        br.src[j] = static_cast<const __half*>(branches_host[j]);
    }
    const int Cy = C5 + nbins * Cb;
    const long long total = set.in_pix[nimg] * (Cy / 8);
    ppm_concat_split_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(set, static_cast<const __half*>(conv5), C5, br, Cb,
                                                                                   static_cast<__half*>(y), Cy);
    RF_LAUNCHED();
    return 0;
}

#define RF_SEG_MAX_CLS 160
#define RF_SEG_MAX_PASSES 8
#define RF_SEG_CPL (RF_SEG_MAX_CLS / 32)           // classes per lane
struct VotePasses { int n, img[RF_SEG_MAX_PASSES]; };

// one warp per output pixel; lane l holds classes l, l + 32, ...  Per pass: bilinear logits, softmax (max, sum of exp, divide),
// scores += p / 5.  A pass that repeats the previous pass's scale reuses its probabilities (the same values the reference recomputes).
__global__ void __launch_bounds__(256) seg_vote_kernel(const __grid_constant__ ImgSet set, const float* __restrict__ logits, int ncls,
                                                       const __grid_constant__ VotePasses vp, int H, int W, int segId, int segFg,
                                                       float* __restrict__ mask, int* __restrict__ cls_out, float* __restrict__ scores_out) {
    const long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pix >= (long long)H * W) return;
    const int Y = (int)(pix / W), X = (int)(pix - (long long)Y * W);
    float score[RF_SEG_CPL], p[RF_SEG_CPL];
#pragma unroll
    for (int q = 0; q < RF_SEG_CPL; ++q) score[q] = p[q] = 0.f;
    int last = -1;
    for (int k = 0; k < vp.n; ++k) {
        const int im = vp.img[k];
        if (im != last) {
            last = im;
            const int h = set.H[im], w = set.W[im];
            int y0, y1, x0, x1;
            float ly0, ly1, lx0, lx1;
            up_coord(Y, h, H, y0, y1, ly0, ly1);
            up_coord(X, w, W, x0, x1, lx0, lx1);
            const float* base = logits + set.in_pix[im] * ncls;
            const float *r00 = base + (long long)(y0 * w + x0) * ncls, *r01 = base + (long long)(y0 * w + x1) * ncls;
            const float *r10 = base + (long long)(y1 * w + x0) * ncls, *r11 = base + (long long)(y1 * w + x1) * ncls;
            float m = -INFINITY;
#pragma unroll
            for (int q = 0; q < RF_SEG_CPL; ++q) {
                const int c = lane + 32 * q;
                p[q] = c < ncls ? up_blend(__ldg(r00 + c), __ldg(r01 + c), __ldg(r10 + c), __ldg(r11 + c), ly0, ly1, lx0, lx1) : -INFINITY;
                m = fmaxf(m, p[q]);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float s = 0.f;
#pragma unroll
            for (int q = 0; q < RF_SEG_CPL; ++q) {
                p[q] = lane + 32 * q < ncls ? expf(p[q] - m) : 0.f;
                s += p[q];
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
#pragma unroll
            for (int q = 0; q < RF_SEG_CPL; ++q) p[q] = __fdiv_rn(p[q], s);
        }
#pragma unroll
        for (int q = 0; q < RF_SEG_CPL; ++q) score[q] = __fadd_rn(score[q], __fdiv_rn(p[q], 5.f));      // segEval.py:36: scores + pred / 5
    }
    // first arg-max: the lane's best (lowest class on ties), then the warp's (pack_key: larger value, then lower index)
    unsigned long long best = 0ull;
#pragma unroll
    for (int q = 0; q < RF_SEG_CPL; ++q) {
        const int c = lane + 32 * q;
        if (c < ncls) {
            const unsigned long long key = pack_key(score[q], (uint32_t)c);
            best = key > best ? key : best;
            if (scores_out) scores_out[pix * ncls + c] = score[q];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other > best ? other : best;
    }
    if (lane == 0) {
        const int pred = (int)key_index(best);
        const float hit = pred == segId ? 1.f : 0.f;
        mask[pix] = segFg ? 1.f - hit : hit;
        if (cls_out) cls_out[pix] = pred;
    }
}

extern "C" int rf_seg_vote(const float* logits, int nimg, const int* hw_host, int ncls, const int* order_host, int norder, int H, int W, int segId,
                           int segFg, float* mask_out, int* class_out, float* scores_out, void* stream) {
    RF_REQUIRE(logits != nullptr && mask_out != nullptr && order_host != nullptr && ncls >= 1 && ncls <= RF_SEG_MAX_CLS && norder >= 1 &&
               norder <= RF_SEG_MAX_PASSES && H >= 1 && W >= 1, "rf_seg_vote: bad arguments (1 <= ncls <= 160, 1 <= norder <= 8)");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 1, 1, 0) == 0, "rf_seg_vote: bad image set");
    VotePasses vp;
    memset(&vp, 0, sizeof(vp));
    vp.n = norder;
    for (int k = 0; k < norder; ++k) {
        RF_REQUIRE(order_host[k] >= 0 && order_host[k] < nimg, "rf_seg_vote: pass order names an image outside the batch");
        vp.img[k] = order_host[k];
    }
    const long long threads = (long long)H * W * 32;
    seg_vote_kernel<<<blocks_for(threads, 256), 256, 0, as_stream(stream)>>>(set, logits, ncls, vp, H, W, segId, segFg, mask_out, class_out, scores_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_l2norm_split_nhwc(const void* x_split, long long P, int C, const uint8_t* mask, float* y, void* y_hi, void* y_lo, void* stream) {
    RF_REQUIRE((C % 8) == 0 && P >= 0, "rf_l2norm_split_nhwc: C must be a multiple of 8");
    RF_REQUIRE(((uintptr_t)x_split % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)y_hi % 16) == 0 && ((uintptr_t)y_lo % 16) == 0,
               "rf_l2norm_split_nhwc: pointers must be 16-byte aligned");
    RF_REQUIRE((y_hi == nullptr) == (y_lo == nullptr), "rf_l2norm_split_nhwc: y_hi and y_lo go together");
    RF_REQUIRE(y != nullptr || y_hi != nullptr, "rf_l2norm_split_nhwc: no output");
    return launch_l2norm<SplitH>(x_split, P, C, mask, y, y_hi, y_lo, stream);
}

extern "C" int rf_corr_neigh_pair_split(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, void* out12_split, void* both_split,
                                        void* stream) {
    RF_REQUIRE((C % 4) == 0 && C <= 1024 && (k % 2) == 1 && ldo >= k * k, "rf_corr_neigh_pair_split: need C % 4 == 0, C <= 1024, odd k, ldo >= k*k");
    RF_REQUIRE(out12_split != nullptr && out12_split != both_split, "rf_corr_neigh_pair_split: outputs");
    return launch_corr_neigh(x, y, N, h, w, C, k, ldo, 3, static_cast<float*>(out12_split), static_cast<float*>(both_split), stream);
}

extern "C" int rf_l2norm_nhwc(const float* x, long long P, int C, const uint8_t* mask, float* y, void* stream) {
    RF_REQUIRE((C % 4) == 0 && P >= 0, "rf_l2norm_nhwc: C must be a multiple of 4");
    return launch_l2norm<float>(x, P, C, mask, y, nullptr, nullptr, stream);
}

extern "C" int rf_corr_neigh_nhwc(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, int round_tf32_out, float* out, void* stream) {
    RF_REQUIRE((C % 4) == 0 && C <= 1024 && (k % 2) == 1 && ldo >= k * k, "rf_corr_neigh_nhwc: need C % 4 == 0, C <= 1024, odd k, ldo >= k*k");
    return launch_corr_neigh(x, y, N, h, w, C, k, ldo, round_tf32_out, out, nullptr, stream);
}

extern "C" int rf_corr_neigh_pair_nhwc(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, int round_tf32_out,
                                       float* out_xy, float* out_yx, void* stream) {
    RF_REQUIRE((C % 4) == 0 && C <= 1024 && (k % 2) == 1 && ldo >= k * k, "rf_corr_neigh_pair_nhwc: need C % 4 == 0, C <= 1024, odd k, ldo >= k*k");
    RF_REQUIRE(out_xy != nullptr && out_yx != nullptr && out_xy != out_yx, "rf_corr_neigh_pair_nhwc: two distinct outputs");
    return launch_corr_neigh(x, y, N, h, w, C, k, ldo, round_tf32_out, out_xy, out_yx, stream);
}

extern "C" int rf_softmax_flow(const float* logits, int N, int h, int w, int k, float* flow_nchw, void* stream) {
    long long P = (long long)N * h * w;
    if (P == 0) return 0;
    softmax_flow_kernel<<<blocks_for(P, 128), 128, 0, as_stream(stream)>>>(logits, N, h, w, k, flow_nchw);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_sigmoid(const float* x, long long n, float* y, void* stream) {
    if (n <= 0) return 0;
    sigmoid_kernel<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(x, n, y);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_preproc_u8(const uint8_t* img, long long npix, int normalize, float* out_nhwc, void* stream) {
    if (npix <= 0) return 0;
    const long long n = npix * 3;
    if (((uintptr_t)img & 3) == 0 && ((uintptr_t)out_nhwc & 15) == 0 && n >= 12) {
        const long long groups = n / 12, tail = n - groups * 12;                 // the tail starts on a pixel boundary too
        preproc_vec_kernel<<<blocks_for(groups, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const unsigned int*>(img), groups, normalize,
                                                                                   reinterpret_cast<float4*>(out_nhwc));
        RF_LAUNCHED();
        if (tail > 0) {
            preproc_kernel<<<1, 32, 0, as_stream(stream)>>>(img + groups * 12, tail, normalize, out_nhwc + groups * 12);
            RF_LAUNCHED();
        }
        return 0;
    }
    preproc_kernel<<<blocks_for(n, 256), 256, 0, as_stream(stream)>>>(img, n, normalize, out_nhwc);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_resample_u8(const uint8_t* in, int in_h, int in_w, int channels, int horizontal,
                              const int* bounds, const int* kk, int ksize, int out_size, uint8_t* out, void* stream) {
    long long total = (long long)(horizontal ? in_h : out_size) * (horizontal ? out_size : in_w) * channels;
    if (total <= 0) return 0;
    if (horizontal) {
        resample_h_kernel<<<blocks_for((long long)in_h * out_size, 256), 256, 0, as_stream(stream)>>>(in, in_h, in_w, channels, bounds, kk, ksize, out_size, out);
        RF_LAUNCHED();
        return 0;
    }
    const long long row_bytes = (long long)in_w * channels;
    if ((row_bytes & 3) == 0 && ((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 3) == 0) {
        resample_v_kernel<<<blocks_for((long long)out_size * (row_bytes >> 2), 256), 256, 0, as_stream(stream)>>>(in, in_h, (int)row_bytes, bounds, kk, ksize, out_size, out);
        RF_LAUNCHED();
        return 0;
    }
    resample_u8_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(in, in_h, in_w, channels, horizontal, bounds, kk, ksize, out_size, out);
    RF_LAUNCHED();
    return 0;
}

// Pillow src/libImaging/Resample.c precompute_coeffs + normalize_coeffs_8bpc for the
// LANCZOS filter (support 3), box = whole image.  Host-side, exact double arithmetic.
static double rf_sinc(double x) {
    if (x == 0.0) return 1.0;
    x = x * 3.14159265358979323846;
    return sin(x) / x;
}
static double rf_lanczos(double x) {
    if (-3.0 <= x && x < 3.0) return rf_sinc(x) * rf_sinc(x / 3);
    return 0.0;
}
static double rf_triangle(double x) {                      // Pillow's bilinear_filter
    if (x < 0.0) x = -x;
    if (x < 1.0) return 1.0 - x;
    return 0.0;
}
// precompute_coeffs + normalize_coeffs_8bpc for a filter of the given support (LANCZOS 3, BILINEAR 1)
static int pil_coeffs_host(double (*filter)(double), double filter_support, int in_size, int out_size, int* bounds_host, int* kk_host,
                           int kk_capacity, int* ksize_out) {
    RF_REQUIRE(in_size > 0 && out_size > 0, "rf_*_coeffs_host: bad sizes");
    double scale, filterscale;
    filterscale = scale = (double)in_size / out_size;
    if (filterscale < 1.0) filterscale = 1.0;
    double support = filter_support * filterscale;
    int ksize = (int)ceil(support) * 2 + 1;
    *ksize_out = ksize;
    if (kk_host == nullptr) return 0;                      // size query
    RF_REQUIRE((long long)ksize * out_size <= kk_capacity, "rf_*_coeffs_host: kk buffer too small");
    double* k = new double[ksize];
    for (int xx = 0; xx < out_size; xx++) {
        double center = 0 + (xx + 0.5) * scale;
        double ww = 0.0;
        double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        int x;
        for (x = 0; x < xmax; x++) {
            double w = filter((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        for (x = 0; x < xmax; x++)
            if (ww != 0.0) k[x] /= ww;
        for (; x < ksize; x++) k[x] = 0;
        bounds_host[xx * 2 + 0] = xmin;
        bounds_host[xx * 2 + 1] = xmax;
        for (x = 0; x < ksize; x++) {
            if (k[x] < 0) kk_host[xx * ksize + x] = (int)(-0.5 + k[x] * (1 << RF_PRECISION_BITS));
            else kk_host[xx * ksize + x] = (int)(0.5 + k[x] * (1 << RF_PRECISION_BITS));
        }
    }
    delete[] k;
    return 0;
}
extern "C" int rf_lanczos_coeffs_host(int in_size, int out_size, int* bounds_host, int* kk_host, int kk_capacity, int* ksize_out) {
    return pil_coeffs_host(rf_lanczos, 3.0, in_size, out_size, bounds_host, kk_host, kk_capacity, ksize_out);
}
extern "C" int rf_bilinear_coeffs_host(int in_size, int out_size, int* bounds_host, int* kk_host, int kk_capacity, int* ksize_out) {
    return pil_coeffs_host(rf_triangle, 1.0, in_size, out_size, bounds_host, kk_host, kk_capacity, ksize_out);
}

extern "C" int rf_warp_grid(const float* H, int N, int h, int w, float* grid_out, void* stream) {
    long long total = (long long)N * h * w;
    if (total <= 0) return 0;
    warp_grid_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(H, N, h, w, grid_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_grid_sample(const float* in, int N, int C, int Hin, int Win, const long long* in_s_host,
                              const float* grid, int Hout, int Wout, int align_corners,
                              float* out, const long long* out_s_host, void* stream) {
    long long total = (long long)N * Hout * Wout;
    if (total <= 0) return 0;
    Strides4 is{in_s_host[0], in_s_host[1], in_s_host[2], in_s_host[3]};
    Strides4 os{out_s_host[0], out_s_host[1], out_s_host[2], out_s_host[3]};
    grid_sample_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(in, N, C, Hin, Win, is, grid, Hout, Wout, align_corners, out, os);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_warp_sample_u8(const float* H, const uint8_t* src, int Hin, int Win, int h, int w, int align_corners, uint8_t* out,
                                 void* stream) {
    RF_REQUIRE(Hin > 0 && Win > 0, "rf_warp_sample_u8: empty source");
    long long total = (long long)h * w;
    if (total <= 0) return 0;
    warp_sample_u8_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(H, src, Hin, Win, h, w, align_corners, out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_affine_sample_u8(const float* theta, const uint8_t* src, int Hin, int Win, int h, int w, float* out_nhwc, void* stream) {
    RF_REQUIRE(Hin > 0 && Win > 0, "rf_affine_sample_u8: empty source");
    long long total = (long long)h * w;
    if (total <= 0) return 0;
    affine_sample_u8_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(theta, src, Hin, Win, h, w, out_nhwc);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_val_keypoints(const float* flowDown8, int h8, int w8, const float* theta, int H, int W, int wA, int hA, const int* kpts,
                                const int* count, int capacity, int pair, const double* thresholds_host, int T, unsigned long long* counts,
                                int* err, double* dist_out, float* flow_out, void* stream) {
    RF_REQUIRE(h8 > 0 && w8 > 0 && H > 0 && W > 0, "rf_val_keypoints: empty flow or target");
    RF_REQUIRE(T >= 1 && T <= RF_VAL_MAX_THRESHOLDS && thresholds_host, "rf_val_keypoints: 1..16 thresholds");
    RF_REQUIRE(counts && err && count, "rf_val_keypoints: counts, error word and count are required");
    if (capacity <= 0) return 0;
    ValThresholds th{};
    for (int t = 0; t < T; ++t) th.t[t] = thresholds_host[t];
    th.n = T;
    val_keypoints_kernel<<<blocks_for(capacity, 256), 256, 0, as_stream(stream)>>>(flowDown8, h8, w8, theta, H, W, wA, hA, kpts, count, capacity,
                                                                                   pair, th, counts, err, dist_out, flow_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_upsample_bilinear(const float* in, int NC, int h, int w, int H, int W, float* out, void* stream) {
    long long total = (long long)NC * H * W;
    if (total <= 0) return 0;
    upsample_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(in, NC, h, w, H, W, out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_compose_fine(const float* flowDown8, const float* match12, const float* match21, int h8, int w8,
                               const float* coarse, int H, int W, int clamp, int align_corners,
                               float* flow12_out, float* match_out, float* flowUp_out, void* stream) {
    long long total = (long long)H * W;
    if (total <= 0) return 0;
    RF_REQUIRE(match_out == nullptr || match12 != nullptr, "rf_compose_fine: match_out needs match12");
    compose_fine_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(flowDown8, match12, match21, h8, w8, coarse, H, W, H, W, clamp,
                                                                              align_corners, flow12_out, match_out, flowUp_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_compose_fine_ex(const float* flowDown8, const float* match12, const float* match21, int h8, int w8,
                                  const float* coarse, int Hc, int Wc, int H, int W, int clamp, int align_corners,
                                  float* flow12_out, float* match_out, float* flowUp_out, void* stream) {
    long long total = (long long)H * W;
    if (total <= 0) return 0;
    RF_REQUIRE(Hc >= 1 && Wc >= 1, "rf_compose_fine_ex: empty coarse grid");
    RF_REQUIRE(match_out == nullptr || match12 != nullptr, "rf_compose_fine_ex: match_out needs match12");
    compose_fine_kernel<<<blocks_for(total, 256), 256, 0, as_stream(stream)>>>(flowDown8, match12, match21, h8, w8, coarse, Hc, Wc, H, W, clamp,
                                                                              align_corners, flow12_out, match_out, flowUp_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" size_t rf_remove_small_cc_workspace(int H, int W) { return 2ull * (size_t)(H > 0 ? H : 0) * (size_t)(W > 0 ? W : 0) * sizeof(int) + 256; }

extern "C" int rf_remove_small_cc(float* match, int N, int H, int W, float match_th, double cc_th, void* ws, size_t ws_bytes, void* stream) {
    if (cc_th == 0.0 || N <= 0 || H <= 0 || W <= 0) return 0;         // evaluation.py:87-88
    RF_REQUIRE((long long)H * W < (1ll << 31), "rf_remove_small_cc: image too large");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_remove_small_cc_workspace(H, W), "rf_remove_small_cc: workspace too small");
    const int n = H * W;
    int* L = reinterpret_cast<int*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    int* cnt = L + n;
    cudaStream_t st = as_stream(stream);
    for (int j = 0; j < N; ++j) {                                     // getResults.py:71 loops over the hypotheses
        float* m = match + (long long)j * n;
        cc_init_kernel<<<blocks_for(n, 256), 256, 0, st>>>(m, match_th, n, L, cnt);
        RF_LAUNCHED();
        cc_merge_kernel<<<blocks_for(n, 256), 256, 0, st>>>(L, H, W);
        RF_LAUNCHED();
        cc_flatten_count_kernel<<<blocks_for(n, 256), 256, 0, st>>>(L, n, cnt);
        RF_LAUNCHED();
        cc_filter_kernel<<<blocks_for(n, 256), 256, 0, st>>>(m, L, cnt, n, cc_th);
        RF_LAUNCHED();
    }
    return 0;
}

extern "C" size_t rf_fill_nearest_matched_workspace(int H, int W) {
    const size_t h = H > 0 ? H : 0, w = W > 0 ? W : 0;
    return 2 * h * w * sizeof(int) + h * (w + 1) * sizeof(double) + 512;
}

extern "C" int rf_fill_nearest_matched(const float* flow, const uint8_t* matched, int H, int W, float* flow_out, int* index_out,
                                       void* ws, size_t ws_bytes, void* stream) {
    if (H <= 0 || W <= 0) return 0;
    RF_REQUIRE(flow != flow_out, "rf_fill_nearest_matched: in-place is not supported");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_fill_nearest_matched_workspace(H, W), "rf_fill_nearest_matched: workspace too small");
    const size_t n = (size_t)H * W;
    double* z = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    int* gy = reinterpret_cast<int*>(z + (size_t)H * (W + 1));
    int* v = gy + n;
    cudaStream_t st = as_stream(stream);
    edt_cols_kernel<<<blocks_for(W, 64), 64, 0, st>>>(matched, H, W, gy);
    RF_LAUNCHED();
    edt_rows_fill_kernel<<<blocks_for(H, 32), 32, 0, st>>>(gy, H, W, v, z, reinterpret_cast<const float2*>(flow),
                                                          reinterpret_cast<float2*>(flow_out), index_out);
    RF_LAUNCHED();
    return 0;
}

// scipy.misc.bytescale(np.rot90(map, rot)) as SciPy 1.2's imresize computes it on a float32 map (the drivers'
// `imresize(It_bg, (h, w)) < 128` before its PIL resize).  Two launches, no host read, so the call can be captured in a CUDA
// graph: (1) every CTA reduces a strided slice of the map to its (min, max); (2) every CTA reduces those partials in one fixed
// order (min / max are exact, so any order gives the same bits) and byte-scales its output pixels in fp32:
//   span = cmax - cmin (1 when 0); scale = 255 / span; v = clip((x - cmin) * scale, 0, 255) + 0.5; out = (uint8)v.
// NaN-free maps only (fminf / fmaxf drop a NaN where numpy propagates it).
#define RF_BYTESCALE_PARTS 256
#define RF_BYTESCALE_THREADS 256

static __device__ __forceinline__ float2 minmax_block(float lo, float hi, float2* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = make_float2(lo, hi);
    __syncthreads();
    if (warp == 0) {
        float2 v = lane < (RF_BYTESCALE_THREADS >> 5) ? red[lane] : make_float2(INFINITY, -INFINITY);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            v.x = fminf(v.x, __shfl_xor_sync(0xffffffffu, v.x, o));
            v.y = fmaxf(v.y, __shfl_xor_sync(0xffffffffu, v.y, o));
        }
        if (lane == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

__global__ void __launch_bounds__(RF_BYTESCALE_THREADS) bytescale_minmax_kernel(const float* __restrict__ x, long long n, float2* __restrict__ part) {
    __shared__ float2 red[RF_BYTESCALE_THREADS / 32];
    float lo = INFINITY, hi = -INFINITY;
    for (long long i = (long long)blockIdx.x * RF_BYTESCALE_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * RF_BYTESCALE_THREADS) {
        const float v = __ldg(x + i);
        lo = fminf(lo, v);
        hi = fmaxf(hi, v);
    }
    const float2 r = minmax_block(lo, hi, red);
    if (threadIdx.x == 0) part[blockIdx.x] = r;
}

// out [Ho][Wo] = bytescale(np.rot90(x [H][W], rot)); rot 1: out[i][j] = x[j][W-1-i], 2: x[H-1-i][W-1-j], 3: x[H-1-j][i]
__global__ void __launch_bounds__(RF_BYTESCALE_THREADS) bytescale_rot_kernel(const float* __restrict__ x, int H, int W, int rot,
                                                                            const float2* __restrict__ part, int nparts, uint8_t* __restrict__ out) {
    __shared__ float2 red[RF_BYTESCALE_THREADS / 32];
    float lo = INFINITY, hi = -INFINITY;
    for (int p = threadIdx.x; p < nparts; p += RF_BYTESCALE_THREADS) {
        const float2 v = part[p];
        lo = fminf(lo, v.x);
        hi = fmaxf(hi, v.y);
    }
    const float2 mm = minmax_block(lo, hi, red);
    const float cmin = mm.x;
    const float span = __fsub_rn(mm.y, mm.x);
    const float scale = span == 0.f ? 255.f : __fdiv_rn(255.f, span);
    const int Ho = (rot & 1) ? W : H, Wo = (rot & 1) ? H : W;
    const long long n = (long long)Ho * Wo;
    for (long long o = (long long)blockIdx.x * RF_BYTESCALE_THREADS + threadIdx.x; o < n; o += (long long)gridDim.x * RF_BYTESCALE_THREADS) {
        const int i = (int)(o / Wo), j = (int)(o - (long long)i * Wo);
        int r, c;
        switch (rot) {
            case 1: r = j; c = W - 1 - i; break;
            case 2: r = H - 1 - i; c = W - 1 - j; break;
            case 3: r = H - 1 - j; c = i; break;
            default: r = i; c = j; break;
        }
        float v = __fmul_rn(__fsub_rn(__ldg(x + (long long)r * W + c), cmin), scale);
        v = fminf(fmaxf(v, 0.f), 255.f);
        out[o] = (uint8_t)(int)__fadd_rn(v, 0.5f);
    }
}

extern "C" size_t rf_bytescale_mask_u8_workspace(int H, int W) {
    (void)H;
    (void)W;
    return RF_BYTESCALE_PARTS * sizeof(float2) + 256;
}

extern "C" int rf_bytescale_mask_u8(const float* map, int H, int W, int rot, uint8_t* out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(map != nullptr && out != nullptr && H >= 1 && W >= 1 && rot >= 0 && rot <= 3,
               "rf_bytescale_mask_u8: need a non-empty map, an output and 0 <= rot <= 3");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_bytescale_mask_u8_workspace(H, W), "rf_bytescale_mask_u8: workspace too small");
    const long long n = (long long)H * W;
    float2* part = reinterpret_cast<float2*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    long long want = (n + 4 * RF_BYTESCALE_THREADS - 1) / (4 * RF_BYTESCALE_THREADS);       // >= 4 elements per thread
    const int nparts = (int)(want < 1 ? 1 : (want > RF_BYTESCALE_PARTS ? RF_BYTESCALE_PARTS : want));
    cudaStream_t st = as_stream(stream);
    bytescale_minmax_kernel<<<nparts, RF_BYTESCALE_THREADS, 0, st>>>(map, n, part);
    RF_LAUNCHED();
    long long blocks = (n + RF_BYTESCALE_THREADS - 1) / RF_BYTESCALE_THREADS;
    if (blocks > 1024) blocks = 1024;
    bytescale_rot_kernel<<<(unsigned)blocks, RF_BYTESCALE_THREADS, 0, st>>>(map, H, W, rot, part, nparts, out);
    RF_LAUNCHED();
    return 0;
}

// One hypothesis of evalKITTI's loop after remove_small_cc (evaluation/evalKITTI/evaluation.py:316-326), with the host's
// decisions turned into a device flag.  Two launches, no host read, no atomics, so the step can be captured in a CUDA graph and
// gives the same bits every run:
//   (1) every CTA counts the pixels of a strided slice with match > 0.9999 and fgMask == 0 (both factors of the reference's
//       `(matchFine > 0.9999) * (1 - fgMask)` are 0 / 1, so the count is exact); block 0 also snapshots the incoming flag;
//   (2) every CTA sums those partials in one fixed order, decides ok = status == 0 && (first || count >= cmin) and
//       alive = alive_in && ok, and where alive holds rewrites its pixels in fp32 exactly as numpy evaluates them:
//       Mask = ((Mask + match * (1 - fgMask)) > 0.9999), then fgMask = ((Mask + (1 - bg)) > 0.5).
// Launch 2 reads the snapshot, never the flag it writes.  A dead hypothesis leaves Mask and fgMask untouched (its match may be
// the NaN of a failed RANSAC's H = 0).
#define RF_KITTI_PARTS 256
#define RF_KITTI_THREADS 256

static __device__ __forceinline__ int sum_block(int v, int* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < (RF_KITTI_THREADS >> 5) ? red[lane] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

__global__ void __launch_bounds__(RF_KITTI_THREADS) kitti_region_count_kernel(const float* __restrict__ match, const float* __restrict__ fg,
                                                                             int n, const int* __restrict__ alive, int* __restrict__ part,
                                                                             int* __restrict__ alive_prev) {
    __shared__ int red[RF_KITTI_THREADS / 32];
    int c = 0;
    for (int i = blockIdx.x * RF_KITTI_THREADS + threadIdx.x; i < n; i += gridDim.x * RF_KITTI_THREADS)
        c += (__ldg(match + i) > 0.9999f && __ldg(fg + i) == 0.f) ? 1 : 0;
    c = sum_block(c, red);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = c;
        if (blockIdx.x == 0) *alive_prev = *alive;
    }
}

__global__ void __launch_bounds__(RF_KITTI_THREADS) kitti_region_update_kernel(const float* __restrict__ match, float* __restrict__ Mask,
                                                                              const float* __restrict__ bg, float* __restrict__ fg, int n,
                                                                              const int* __restrict__ status, const int* __restrict__ alive_prev,
                                                                              const int* __restrict__ part, int nparts, int first, int cmin,
                                                                              int* __restrict__ alive, int* __restrict__ rec) {
    __shared__ int red[RF_KITTI_THREADS / 32];
    int c = 0;
    for (int p = threadIdx.x; p < nparts; p += RF_KITTI_THREADS) c += part[p];
    const int count = sum_block(c, red);
    const bool live = *alive_prev != 0 && *status == 0 && (first || count >= cmin);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *alive = live ? 1 : 0;
        if (rec != nullptr) {
            rec[0] = live ? 1 : 0;
            rec[1] = count;
        }
    }
    if (!live) return;
    for (int i = blockIdx.x * RF_KITTI_THREADS + threadIdx.x; i < n; i += gridDim.x * RF_KITTI_THREADS) {
        const float f = fg[i];
        const float m = __fadd_rn(Mask[i], __fmul_rn(__ldg(match + i), __fsub_rn(1.f, f))) > 0.9999f ? 1.f : 0.f;
        Mask[i] = m;
        fg[i] = __fadd_rn(m, __fsub_rn(1.f, __ldg(bg + i))) > 0.5f ? 1.f : 0.f;
    }
}

extern "C" size_t rf_kitti_region_step_workspace(int H, int W) {
    (void)H;
    (void)W;
    return RF_KITTI_PARTS * sizeof(int) + 2 * 256;
}

extern "C" int rf_kitti_region_step(const float* match, float* Mask, const float* bg, float* fgMask, int H, int W, const int* status,
                                    int* alive, int first, int cmin, int* rec, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(match != nullptr && Mask != nullptr && bg != nullptr && fgMask != nullptr && status != nullptr && alive != nullptr &&
               H >= 1 && W >= 1, "rf_kitti_region_step: need non-empty maps, a status and an alive flag");
    RF_REQUIRE((long long)H * W < (1ll << 31), "rf_kitti_region_step: map too large");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_kitti_region_step_workspace(H, W), "rf_kitti_region_step: workspace too small");
    const int n = H * W;
    int* part = reinterpret_cast<int*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    int* alive_prev = part + RF_KITTI_PARTS;
    const int want = (n + 4 * RF_KITTI_THREADS - 1) / (4 * RF_KITTI_THREADS);       // >= 4 pixels per thread
    const int nparts = want < 1 ? 1 : (want > RF_KITTI_PARTS ? RF_KITTI_PARTS : want);
    cudaStream_t st = as_stream(stream);
    kitti_region_count_kernel<<<nparts, RF_KITTI_THREADS, 0, st>>>(match, fgMask, n, alive, part, alive_prev);
    RF_LAUNCHED();
    int blocks = (n + RF_KITTI_THREADS - 1) / RF_KITTI_THREADS;
    if (blocks > 1024) blocks = 1024;
    kitti_region_update_kernel<<<blocks, RF_KITTI_THREADS, 0, st>>>(match, Mask, bg, fgMask, n, status, alive_prev, part, nparts, first,
                                                                   cmin, alive, rec);
    RF_LAUNCHED();
    return 0;
}
