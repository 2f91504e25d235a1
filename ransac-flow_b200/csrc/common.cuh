// Shared helpers for the ransacflow_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/ransacflow_b200.h"

namespace rf {

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

inline int fail(const char* what, cudaError_t e, const char* file, int line) {
    snprintf(g_err, sizeof(g_err), "%s: %s (%s:%d)", what, cudaGetErrorString(e), file, line);
    return 1;
}
inline int fail_msg(const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return 2;
}

#define RF_CUDA(expr)                                                   \
    do {                                                                \
        cudaError_t _e = (expr);                                        \
        if (_e != cudaSuccess) return rf::fail(#expr, _e, __FILE__, __LINE__); \
    } while (0)

// call after every kernel launch: counts the launch and surfaces launch errors
#define RF_LAUNCHED()                                                   \
    do {                                                                \
        rf::g_launches.fetch_add(1, std::memory_order_relaxed);         \
        cudaError_t _e = cudaGetLastError();                            \
        if (_e != cudaSuccess) return rf::fail("kernel launch", _e, __FILE__, __LINE__); \
    } while (0)

#define RF_REQUIRE(cond, msg)                                           \
    do {                                                                \
        if (!(cond)) return rf::fail_msg(msg " [" #cond "]");           \
    } while (0)

// engine 4: eight fp32 values as a split tensor's hi / lo planes (`plane` elements apart), clamped to the fp16 range:
// hi = fp16(x), lo = fp16((x - hi) * 2^11).  Shared by the pooling / blur kernels and the fused stem + max-pool.
__device__ __forceinline__ void split_store8(__half* p, long long plane, const float (&v)[8]) {
    uint4 th, tl;
    __half2* h = reinterpret_cast<__half2*>(&th);
    __half2* l = reinterpret_cast<__half2*>(&tl);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float a = fminf(fmaxf(v[2 * e], -65504.f), 65504.f), b = fminf(fmaxf(v[2 * e + 1], -65504.f), 65504.f);
        h[e] = __floats2half2_rn(a, b);
        const float2 f = __half22float2(h[e]);
        l[e] = __floats2half2_rn((a - f.x) * 2048.f, (b - f.y) * 2048.f);
    }
    *reinterpret_cast<uint4*>(p) = th;
    *reinterpret_cast<uint4*>(p + plane) = tl;
}
inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < 64) ? dev : 0;
}

inline int num_sms() {
    static int n[64] = {0};
    const int dev = current_device();
    if (n[dev] == 0) {
        cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
        if (n[dev] <= 0) n[dev] = 132;
    }
    return n[dev];
}

// ragged NHWC batch descriptor passed by value to kernels
struct ImgSet {
    int n;
    int H[RF_MAX_IMGS], W[RF_MAX_IMGS];
    int Ho[RF_MAX_IMGS], Wo[RF_MAX_IMGS];
    long long in_pix[RF_MAX_IMGS + 1];    // prefix sums of H*W   (pixel offsets of each image in x)
    long long out_pix[RF_MAX_IMGS + 1];   // prefix sums of Ho*Wo (pixel offsets of each image in y)
};

inline int make_imgset(ImgSet& s, int nimg, const int* hw, int k, int stride, int pad) {
    if (nimg < 1 || nimg > RF_MAX_IMGS) return 1;
    s.n = nimg;
    s.in_pix[0] = 0;
    s.out_pix[0] = 0;
    for (int i = 0; i < nimg; ++i) {
        s.H[i] = hw[2 * i];
        s.W[i] = hw[2 * i + 1];
        s.Ho[i] = (s.H[i] + 2 * pad - k) / stride + 1;
        s.Wo[i] = (s.W[i] + 2 * pad - k) / stride + 1;
        if (s.Ho[i] < 1 || s.Wo[i] < 1) return 1;
        s.in_pix[i + 1] = s.in_pix[i] + (long long)s.H[i] * s.W[i];
        s.out_pix[i + 1] = s.out_pix[i] + (long long)s.Ho[i] * s.Wo[i];
    }
    for (int i = nimg; i < RF_MAX_IMGS; ++i) {
        s.H[i] = s.W[i] = s.Ho[i] = s.Wo[i] = 0;
        s.in_pix[i + 1] = s.in_pix[nimg];
        s.out_pix[i + 1] = s.out_pix[nimg];
    }
    return 0;
}

struct ConvParams {
    const float* x;
    const float* w;          // [R*S*Cin][Cout]
    const float* bias;       // nullable
    const float* residual;   // nullable, packed like y
    float* y;
    int Cin, Cout, R, S, stride, pad, relu;
    int round_out;           // 1: round the output to TF32 (nearest) so that the tensor-core consumer's truncation is exact
    int dil;                 // tap spacing (1 = none; > 1 only on the split engine)
    long long Mtot;          // total output pixels
    int K;                   // R*S*Cin
};

// locate the image a packed output pixel belongs to
__device__ __forceinline__ int find_img(const ImgSet& s, long long p) {
    int i = 0;
#pragma unroll
    for (int j = 1; j < RF_MAX_IMGS; ++j) i += (j < s.n && p >= s.out_pix[j]) ? 1 : 0;
    return i;
}

// monotone float -> uint32 map (larger float <=> larger unsigned)
__device__ __forceinline__ uint32_t f2ord(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// round-to-nearest TF32 (10-bit mantissa); the tensor core itself truncates fp32 operands
__device__ __forceinline__ float round_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float ord2f(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
// (value, index) -> 64-bit key: max over keys = max value, ties -> smallest index
__device__ __forceinline__ unsigned long long pack_key(float v, uint32_t idx) {
    return ((unsigned long long)f2ord(v) << 32) | (unsigned long long)(0xFFFFFFFFu - idx);
}
__device__ __forceinline__ uint32_t key_index(unsigned long long k) { return 0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull); }
__device__ __forceinline__ float key_value(unsigned long long k) { return ord2f((uint32_t)(k >> 32)); }

}  // namespace rf
