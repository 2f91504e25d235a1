// Tensor-core engine (sm_90a): implicit-GEMM convolutions and the correlation with its row / column arg-max, on wgmma.
//
// One kernel template.  An output tile is 128 pixels (correlation: 128 rows of featA) x BN channels (columns of featB); the
// pixels are a tw x (128 / tw) rectangle of one image, or for 1x1 / stride-1 layers 128 consecutive pixels of the batch (flat
// tiles, see conv_impl).  A CTA has 288 threads:
//   warp 8        : TMA producer.  A = box (channels, tw, th[, 2 planes]) of the NHWC image at the tap's offset (out-of-bounds
//                   zero fill is the zero padding, the traversal stride is the convolution stride), B = box of the K-major
//                   weight matrix; both 128-byte swizzled, completion counted on the stage's mbarrier.
//   warpgroups 0-1: tile rows 0..63 / 64..127.  wgmma.mma_async from the stage's descriptors into register accumulators; one
//                   wgmma group stays in flight while the stage before it is handed back to the producer.  The epilogue
//                   works on the registers: bias, residual, ReLU, conversion, store (convolution) or arg-max keys (correlation).
// Convolutions are persistent: tile t (N tiles fastest) runs on CTA t mod gridDim.x, and the ring runs on across tile
// boundaries, so one tile's epilogue overlaps the loads of the next.  fp16 and split outputs take one more ring stage per tile
// (the epilogue slot): the producer TMA-loads the residual tile into it, the consumers add it and write the result back in
// place, one thread TMA-stores the slot and hands it back once the store has read it.  fp32 outputs (rows of 49 or 1 floats
// are not 16-byte multiples) keep register stores.  The correlation runs one tile per CTA.
// Operand kinds:
//   K_TF32   : fp32 operands, TF32 MMAs (engine 1);
//   K_F16    : fp16 operands (engines 2 and 3);
//   K_SPLIT  : every operand as two fp16 planes, x = hi + lo * 2^-11 (22 significand bits, engines 4 / 5 and correlation
//              precision 2): main += hi*hi, cross += lo*hi + hi*lo at 2^11 scale, result = main + cross * 2^-11;
//   K_TF32X3 : fp32 operands split into TF32 hi + lo (correlation precision 1): lo*hi + hi*lo + hi*hi into one accumulator.
#include <cuda.h>
#include <cuda_fp16.h>

#include <climits>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "tc_common.cuh"

namespace rf {

constexpr int K_TF32 = 0, K_F16 = 1, K_SPLIT = 2, K_TF32X3 = 3;
constexpr int MODE_CONV = 0, MODE_CORR = 1;
constexpr int O_F32 = 0, O_F16 = 1, O_SPLIT = 2;     // convolution output (and residual) formats
constexpr int WG_THREADS = 288;                       // two consumer warpgroups + the producer warp

struct alignas(64) WgParams {
    CUtensorMap mapA[RF_MAX_IMGS];        // per image: input (C, W, H[, 2]); correlation: A hi (C, NA, 1)
    CUtensorMap mapA2[RF_MAX_IMGS];       // dual-input 1x1: the second input (Cin2, W2, H2, 2); correlation: [0] = A lo
    CUtensorMap mapY[RF_MAX_IMGS];        // fp16 / split output per image: (Cout, Wo, Ho[, 2]), box (64, tw, th[, 2])
    CUtensorMap mapR[RF_MAX_IMGS];        // its residual, same geometry
    CUtensorMap mapB;                     // weights (K, Cout[, 2]); correlation: B hi (C, NB)
    CUtensorMap mapBlo;                   // correlation: B lo
    int nimg;
    int ntiles;                           // convolution: pixel tiles of the batch x N tiles
    int tile_start[RF_MAX_IMGS + 1];      // prefix sums of pixel tiles per image
    int tiles_x[RF_MAX_IMGS];
    int tw[RF_MAX_IMGS];                  // tile width (tile height = 128 / tw)
    int Ho[RF_MAX_IMGS], Wo[RF_MAX_IMGS];
    long long out_pix[RF_MAX_IMGS + 1];
    int R, S, pad, stride, Cin, Cout, relu, round_out;
    int dil;                              // tap spacing of a dilated 3x3 (1 otherwise)
    int kc1, stride2;                    // dual-input 1x1: K blocks [0, kc1) come from mapA, the rest from mapA2 (sampled with stride2)
    long long plane;                      // split output / residual: elements from the hi to the lo plane
    const float* bias;
    const void* residual;
    void* y;
    unsigned long long* rowbest;          // correlation
    unsigned long long* colbest;
    int NA, NB;
};
static_assert(sizeof(WgParams) <= 32764, "kernel parameter space (CUDA 12.1+ large kernel parameters)");

template <int KIND, int BN, int MODE>
struct WgCfg {
    static constexpr int NPL = (KIND == K_SPLIT || KIND == K_TF32X3) ? 2 : 1;     // operand planes
    static constexpr int A_BYTES = NPL * TC_A_BYTES;
    static constexpr int B_PLANE = BN * 128;
    static constexpr int STAGE_BYTES = A_BYTES + NPL * B_PLANE;
    // two CTAs per SM (one tile's epilogue overlaps the other's main loop) where the stages and the accumulators allow it
    static constexpr bool ONE_CTA = MODE == MODE_CORR || NPL * BN >= 256;
    static constexpr int BUDGET = ONE_CTA ? 200 * 1024 : 100 * 1024;
    static constexpr int STAGES = BUDGET / STAGE_BYTES > 6 ? 6 : BUDGET / STAGE_BYTES;
    static constexpr int CTAS_PER_SM = ONE_CTA ? 1 : 2;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(STAGES >= 2 && SMEM_BYTES <= 227 * 1024, "shared memory");
};

// fp32 pair -> fp16 pair, saturating at +-65504 instead of overflowing to inf
__device__ __forceinline__ __half2 pack_sat(float a, float b) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));     // first source -> upper half
    return *reinterpret_cast<__half2*>(&r);
}
// (a, b) -> hi = fp16(x), lo = fp16((x - hi) * 2^11), saturating like the fp16 engine
__device__ __forceinline__ void split2(float a, float b, __half2& hi, __half2& lo) {
    hi = pack_sat(a, b);
    const float2 f = __half22float2(hi);
    lo = pack_sat((a - f.x) * 2048.f, (b - f.y) * 2048.f);
}

// One K block (128 bytes of every operand row) of this warpgroup's 64 rows.
template <int KIND, int BN, int NACC>
__device__ __forceinline__ void mma_block(float (&acc)[NACC][BN / 2], uint32_t sa, uint32_t sb) {
    constexpr bool TF32 = KIND == K_TF32 || KIND == K_TF32X3;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t ah = wg_desc(sa + 32 * k), bh = wg_desc(sb + 32 * k);
        if constexpr (KIND == K_SPLIT || KIND == K_TF32X3) {
            const uint64_t al = wg_desc(sa + TC_A_BYTES + 32 * k), bl = wg_desc(sb + BN * 128 + 32 * k);
            float (&x)[BN / 2] = acc[NACC - 1];
            wgmma<TF32, BN>(x, al, bh);
            wgmma<TF32, BN>(x, ah, bl);
            wgmma<TF32, BN>(acc[0], ah, bh);
        } else {
            wgmma<TF32, BN>(acc[0], ah, bh);
        }
    }
}

template <int KIND, int BN, int MODE, int OUT>
__global__ void __launch_bounds__(WG_THREADS, WgCfg<KIND, BN, MODE>::CTAS_PER_SM)
wg_kernel(const __grid_constant__ WgParams p) {
    using Cfg = WgCfg<KIND, BN, MODE>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int BK = (KIND == K_TF32 || KIND == K_TF32X3) ? TC_BK : TC_BK_F16;
    constexpr int NACC = KIND == K_SPLIT ? 2 : 1;
    // fp16 / split convolution outputs: epilogue slot + TMA store.  One 64-channel box of the output tile is 128 pixel rows of
    // 128 bytes per plane, swizzled like the operand tiles; the BN / 64 boxes of a tile fit one stage in every instance.
    constexpr bool SLOT = MODE == MODE_CONV && OUT != O_F32;
    constexpr int BOX_BYTES = (OUT == O_SPLIT ? 2 : 1) * 128 * 128;
    static_assert(!SLOT || (BN / 64) * BOX_BYTES <= Cfg::STAGE_BYTES, "the output tile fits one stage");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kc = p.Cin / BK;
    const int KI = p.R * p.S * kc;

    // ---- tiles.  Convolution: tile t -> N tile t % nt, pixel tile t / nt, on CTA t mod gridDim.x: the N tiles of a pixel tile run
    // on neighbouring CTAs at the same time, so its A boxes come from HBM once and from L2 for the other N tiles.  Correlation: one
    // tile per CTA, column tiles fastest, so that the CTAs sharing a 128-row slab of featA run together ----
    const int t_first = MODE == MODE_CORR ? 0 : (int)blockIdx.x;
    const int t_step = MODE == MODE_CORR ? 1 : (int)gridDim.x;
    const int t_end = MODE == MODE_CORR ? 1 : p.ntiles;
    const int nt = (p.Cout + BN - 1) / BN;
    struct Tile { int img, tw, ox0, oy0, n0; };
    auto decode = [&](int t) {
        const int mtile = MODE == MODE_CORR ? (int)blockIdx.y : t / nt;
        const int ntile = MODE == MODE_CORR ? (int)blockIdx.x : t - mtile * nt;
        Tile T;
        T.img = 0;
#pragma unroll
        for (int j = 1; j < RF_MAX_IMGS; ++j) T.img += (j < p.nimg && mtile >= p.tile_start[j]) ? 1 : 0;
        const int tloc = mtile - p.tile_start[T.img];
        T.tw = p.tw[T.img];
        const int tyi = tloc / p.tiles_x[T.img], txi = tloc - tyi * p.tiles_x[T.img];
        T.ox0 = txi * T.tw;
        T.oy0 = tyi * (128 / T.tw);
        T.n0 = ntile * BN;
        return T;
    };
    // 64-channel boxes of the tile that hold output channels (BN = 128 with Cout - n0 <= 64: the second box is all outside)
    auto boxes = [&](const Tile& T) { return BN == 64 || T.n0 + 64 >= p.Cout ? 1 : 2; };

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        // =============================== TMA producer ===============================
        if (lane == 0) {
            tma_prefetch_desc(&p.mapB);
            uint32_t prefetched = 0;              // images whose tensor maps have been prefetched
            int st = 0;
            uint32_t ph = 0;
            for (int t = t_first; t < t_end; t += t_step) {
                const Tile T = decode(t);
                if (!((prefetched >> T.img) & 1u)) {
                    prefetched |= 1u << T.img;
                    tma_prefetch_desc(&p.mapA[T.img]);
                    if constexpr (SLOT) {
                        tma_prefetch_desc(&p.mapY[T.img]);
                        if (p.residual) tma_prefetch_desc(&p.mapR[T.img]);
                    }
                }
                for (int it = 0; it < KI; ++it) {
                    mbar_wait(&empty[st], ph ^ 1);
                    uint8_t* sa = smem + st * Cfg::STAGE_BYTES;
                    uint8_t* sb = sa + Cfg::A_BYTES;
                    mbar_expect_tx(&full[st], Cfg::STAGE_BYTES);
                    if constexpr (MODE == MODE_CORR) {
                        const int c0 = it * BK;
                        tma_load_3d(sa, &p.mapA[0], &full[st], c0, T.ox0, 0);
                        tma_load_3d(sa + TC_A_BYTES, &p.mapA2[0], &full[st], c0, T.ox0, 0);
                        tma_load_2d(sb, &p.mapB, &full[st], c0, T.n0);
                        tma_load_2d(sb + Cfg::B_PLANE, &p.mapBlo, &full[st], c0, T.n0);
                    } else {
                        const int tap = it / kc, cc = it - tap * kc;
                        const int r = tap / p.S, s = tap - r * p.S;
                        // dilated taps: boxes wholly or partly outside the image are zero-filled by TMA, which is the padding
                        const int c0 = cc * BK, x = T.ox0 * p.stride + s * p.dil - p.pad, y = T.oy0 * p.stride + r * p.dil - p.pad;
                        const int kcol = tap * p.Cin + c0;
                        if constexpr (KIND == K_SPLIT) {       // one 4-D box brings [hi tile | lo tile]
                            if (cc < p.kc1) tma_load_4d(sa, &p.mapA[T.img], &full[st], c0, x, y, 0);
                            else tma_load_4d(sa, &p.mapA2[T.img], &full[st], (cc - p.kc1) * BK, T.ox0 * p.stride2, T.oy0 * p.stride2, 0);
                            tma_load_3d(sb, &p.mapB, &full[st], kcol, T.n0, 0);
                        } else {
                            tma_load_3d(sa, &p.mapA[T.img], &full[st], c0, x, y);
                            tma_load_2d(sb, &p.mapB, &full[st], kcol, T.n0);
                        }
                    }
                    if (++st == STAGES) { st = 0; ph ^= 1; }
                }
                if constexpr (SLOT) {                  // the epilogue slot: the residual tile, or just the hand-over
                    mbar_wait(&empty[st], ph ^ 1);
                    if (p.residual) {
                        const int nb = boxes(T);
                        uint8_t* slot = smem + st * Cfg::STAGE_BYTES;
                        mbar_expect_tx(&full[st], nb * BOX_BYTES);
                        for (int b = 0; b < nb; ++b) {
                            if constexpr (OUT == O_SPLIT) tma_load_4d(slot + b * BOX_BYTES, &p.mapR[T.img], &full[st], T.n0 + 64 * b, T.ox0, T.oy0, 0);
                            else tma_load_3d(slot + b * BOX_BYTES, &p.mapR[T.img], &full[st], T.n0 + 64 * b, T.ox0, T.oy0);
                        }
                    } else {
                        mbar_arrive(&full[st]);
                    }
                    if (++st == STAGES) { st = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // =============================== consumers: warpgroup g owns tile rows 64g .. 64g + 63 ===============================
    const int g = warp >> 2;
    // accumulator fragment: d[4j + 2h + e] = row 16 * (warp % 4) + lane / 4 + 8h, column 8j + 2 * (lane % 4) + e
    const int rbase = 64 * g + 16 * (warp & 3) + (lane >> 2);
    const int cbase = 2 * (lane & 3);
    auto before = [](int s) { return s == 0 ? STAGES - 1 : s - 1; };
    int st = 0;
    uint32_t ph = 0;
    bool stored = false;                          // the stage before `st` is an epilogue slot a TMA store may still be reading
    for (int t = t_first; t < t_end; t += t_step) {
        const Tile T = decode(t);
        float acc[NACC][BN / 2];
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[a][i] = 0.f;
        for (int it = 0; it < KI; ++it) {
            mbar_wait(&full[st], ph);
            const uint32_t sa = smem_u32(smem + st * Cfg::STAGE_BYTES);
            wg_fence();
            mma_block<KIND, BN, NACC>(acc, sa + g * (64 * 128), sa + Cfg::A_BYTES);
            wg_commit();
            wg_wait<1>();                         // the previous stage's MMAs are done: hand it back
            if (it > 0) {
                mbar_arrive(&empty[before(st)]);
            } else if (SLOT && stored) {          // the previous tile's slot, once its store has read it
                if (threadIdx.x == 0) bulk_wait_read();
                mbar_arrive(&empty[before(st)]);
            }
            if (++st == STAGES) { st = 0; ph ^= 1; }
        }
        wg_wait<0>();
#pragma unroll
        for (int a = 0; a < NACC; ++a) wg_fence_regs(acc[a]);
        mbar_arrive(&empty[before(st)]);         // the tile's last K block

        auto value = [&](int i) -> float {
            if constexpr (KIND == K_SPLIT) return fmaf(acc[1][i], 0.00048828125f, acc[0][i]);
            else return acc[0][i];
        };

        if constexpr (SLOT) {
            // element (pixel m, channel c) of the tile: box c / 64, row m, 16-byte chunk ((c % 64) / 8) ^ (m % 8); lo plane
            // 128 rows further.  Each thread reads its residual elements and overwrites them with its outputs.
            mbar_wait(&full[st], ph);
            uint8_t* slot = smem + st * Cfg::STAGE_BYTES;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = rbase + 8 * h;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = 8 * j + cbase, n = T.n0 + c;
                    if (n >= p.Cout) continue;    // Cout % 8 == 0: both channels of the pair exist
                    float v0 = value(4 * j + 2 * h), v1 = value(4 * j + 2 * h + 1);
                    if (p.bias) { v0 += __ldg(p.bias + n); v1 += __ldg(p.bias + n + 1); }
                    uint8_t* e = slot + (c >> 6) * BOX_BYTES + m * 128 + ((((c & 63) >> 3) ^ (m & 7)) << 4) + (c & 7) * 2;
                    if (p.residual) {
                        if constexpr (OUT == O_F16) {
                            const float2 r = __half22float2(*reinterpret_cast<const __half2*>(e));
                            v0 += r.x; v1 += r.y;
                        } else {
                            const float2 rh = __half22float2(*reinterpret_cast<const __half2*>(e));
                            const float2 rl = __half22float2(*reinterpret_cast<const __half2*>(e + 128 * 128));
                            v0 += fmaf(rl.x, 0.00048828125f, rh.x); v1 += fmaf(rl.y, 0.00048828125f, rh.y);
                        }
                    }
                    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    if constexpr (OUT == O_F16) {
                        *reinterpret_cast<__half2*>(e) = pack_sat(v0, v1);
                    } else {
                        __half2 hi, lo;
                        split2(v0, v1, hi, lo);
                        *reinterpret_cast<__half2*>(e) = hi;
                        *reinterpret_cast<__half2*>(e + 128 * 128) = lo;
                    }
                }
            }
            fence_proxy_async();                  // the generic-proxy writes -> visible to the TMA store
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (threadIdx.x == 0) {
                const int nb = boxes(T);
                for (int b = 0; b < nb; ++b) {
                    if constexpr (OUT == O_SPLIT) tma_store_4d(&p.mapY[T.img], slot + b * BOX_BYTES, T.n0 + 64 * b, T.ox0, T.oy0, 0);
                    else tma_store_3d(&p.mapY[T.img], slot + b * BOX_BYTES, T.n0 + 64 * b, T.ox0, T.oy0);
                }
                bulk_commit();
            }
            stored = true;
            if (++st == STAGES) { st = 0; ph ^= 1; }
        } else if constexpr (MODE == MODE_CONV) {
            const int img = T.img, tw = T.tw;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = rbase + 8 * h;
                const int py = m / tw, px = m - py * tw;
                const int oy = T.oy0 + py, ox = T.ox0 + px;
                if (oy >= p.Ho[img] || ox >= p.Wo[img]) continue;
                const long long pix = p.out_pix[img] + (long long)oy * p.Wo[img] + ox;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int n = T.n0 + 8 * j + cbase;
                    if (n >= p.Cout) continue;
                    const bool two = n + 1 < p.Cout;
                    float v0 = value(4 * j + 2 * h), v1 = value(4 * j + 2 * h + 1);
                    if (p.bias) { v0 += __ldg(p.bias + n); if (two) v1 += __ldg(p.bias + n + 1); }
                    const long long o = pix * p.Cout + n;
                    if (p.residual) {
                        const float* r = static_cast<const float*>(p.residual) + o;
                        v0 += __ldg(r); if (two) v1 += __ldg(r + 1);
                    }
                    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    if (p.round_out) { v0 = round_tf32(v0); v1 = round_tf32(v1); }
                    float* y = static_cast<float*>(p.y) + o;
                    if (two && (p.Cout & 1) == 0) *reinterpret_cast<float2*>(y) = make_float2(v0, v1);
                    else { y[0] = v0; if (two) y[1] = v1; }
                }
            }
        } else {
            // utils/outil.py:36-37: per row the best (score, smallest column) key, per column the best (score, smallest row) key.
            // Rows: the four lanes of a quad share a row.  Columns: the eight row groups of a warp by shuffles, then the eight
            // warps through shared memory (the stages are idle: every TMA load has been consumed).
            const int n0 = T.n0;
            unsigned long long* sCol = reinterpret_cast<unsigned long long*>(smem);       // [8 warps][BN]
            const int row0 = T.ox0 + rbase, row1 = row0 + 8;
            const bool rv0 = row0 < p.NA, rv1 = row1 < p.NA;
            unsigned long long rb0 = 0ull, rb1 = 0ull;
            asm volatile("bar.sync 1, 256;" ::: "memory");          // both warpgroups are past their last wgmma reads
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = 8 * j + cbase + e, col = n0 + c;
                    const bool cv = col < p.NB;
                    const float s0 = value(4 * j + e), s1 = value(4 * j + 2 + e);
                    unsigned long long ck = 0ull;
                    if (cv) {
                        if (rv0) { const unsigned long long k = pack_key(s0, (uint32_t)col); rb0 = k > rb0 ? k : rb0; ck = pack_key(s0, (uint32_t)row0); }
                        if (rv1) { const unsigned long long k = pack_key(s1, (uint32_t)col); rb1 = k > rb1 ? k : rb1;
                                   const unsigned long long k1 = pack_key(s1, (uint32_t)row1); ck = k1 > ck ? k1 : ck; }
                    }
#pragma unroll
                    for (int off = 4; off < 32; off <<= 1) {
                        const unsigned long long o = __shfl_xor_sync(0xffffffffu, ck, off);
                        ck = o > ck ? o : ck;
                    }
                    if (lane < 4) sCol[warp * BN + c] = ck;
                }
            }
#pragma unroll
            for (int off = 1; off < 4; off <<= 1) {
                const unsigned long long o0 = __shfl_xor_sync(0xffffffffu, rb0, off), o1 = __shfl_xor_sync(0xffffffffu, rb1, off);
                rb0 = o0 > rb0 ? o0 : rb0;
                rb1 = o1 > rb1 ? o1 : rb1;
            }
            if ((lane & 3) == 0) {
                if (rv0 && rb0 != 0ull) atomicMax(p.rowbest + row0, rb0);
                if (rv1 && rb1 != 0ull) atomicMax(p.rowbest + row1, rb1);
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            for (int c = threadIdx.x; c < BN; c += 256) {
                if (n0 + c >= p.NB) continue;
                unsigned long long cb = 0ull;
#pragma unroll
                for (int w = 0; w < 8; ++w) { const unsigned long long k = sCol[w * BN + c]; cb = k > cb ? k : cb; }
                if (cb != 0ull) atomicMax(p.colbest + n0 + c, cb);
            }
        }
    }
    if constexpr (SLOT)
        if (threadIdx.x == 0) bulk_wait();        // the last tile's stores complete before the CTA (and its shared memory) goes
}


// ------------------------------------------------------------------------------------------------------------
// ResNet-50 front end, fused: conv 7x7 / stride 2 / pad 3 on the 3-channel fp32 image + folded BN + ReLU and, with pool = 1,
// the 3x3 / stride 2 / pad 1 max-pool on its output -> fp16 (engine 2) or split (engine 4) NHWC.  No im2col matrix goes to
// HBM, and with pool = 1 neither does the full-resolution stem output.
// Persistent, 256 threads, 1 CTA per SM: the weights are TMA-loaded once per CTA and stay resident.  A work unit (step) is a
// tile of 4 stem rows x 32 stem columns (128 pixels x 64 channels); units run down column strips (steps fastest) and CTA b
// takes the contiguous range [U b / G, U (b + 1) / G) of them.  Per step:
//   build    : two threads per pixel build its 147-long (r, s, c) patch from the staged 13 x 69 x 3 input window (split into
//              (hi, lo) pairs once, at staging) as hi / lo planes in the 128-byte-swizzled K-major layout (3 K blocks of 64;
//              147..191 are zeros); K block kb + 1 is built while the wgmmas of K block kb run;
//   MMA      : warpgroup g = pixels 64g .. 64g + 63, wgmma over the three K blocks against the resident weights;
//   prefetch : while the MMAs run, the next step's input window is loaded into registers (staged after the MMAs);
//   epilogue : pool = 0: bias, ReLU, conversion and stores from the registers.  pool = 1: the stem values go to a shared tile
//              (engine 4: split and rebuilt, i.e. the values the max-pool of a split tensor reads), then the step's 2 pooled
//              rows x 15 pooled columns are reduced there and stored with 16-byte stores.
// Pooling: pooled column q needs stem columns 2q - 1 .. 2q + 1, so the tiles of strip s start at stem column 30 s - 1 and
// overlap the strip to their left by one column (1/16 of the stem is computed twice); pooled row p needs stem rows
// 2p - 1 .. 2p + 1, so each step keeps its last stem row for the next step of the strip (two alternating tiles).  A CTA whose
// range starts inside a strip first computes the step above, without pooling it.  As in the standalone max-pool, window
// positions outside the stem image are skipped and the maximum runs over (r, s) in the same order.
// ------------------------------------------------------------------------------------------------------------
constexpr int ST_TW = 32, ST_TH = 4, ST_K = 7, ST_C = 3, ST_KK = 147, ST_KB = 3;
constexpr int ST_PW = (ST_TW - 2) / 2, ST_PH = ST_TH / 2;                // pooled columns per strip, pooled rows per step
constexpr int ST_IN_W = ((ST_TW - 1) * 2 + ST_K) * ST_C;                  // 207 floats per staged input row
constexpr int ST_IN_H = (ST_TH - 1) * 2 + ST_K;                           // 13 rows
constexpr int ST_IN_LD = 208;
constexpr int ST_THREADS = 256;
constexpr int ST_B_PLANE = 64 * 128;                                      // one K block of 64 weight rows: 8 KB
constexpr int ST_OFF_ALO = ST_KB * TC_A_BYTES;                            // 48 KB: lo planes of the patches
constexpr int ST_OFF_B = 2 * ST_KB * TC_A_BYTES;                          // 96 KB
constexpr int ST_OFF_T = ST_OFF_B + ST_KB * 2 * ST_B_PLANE;               // 144 KB: two stem tiles of 128 pixels x 64 fp32
constexpr int ST_T_BYTES = 128 * 64 * 4;
constexpr int ST_OFF_IN = ST_OFF_T + 2 * ST_T_BYTES;                      // 208 KB
constexpr int ST_OFF_BAR = ST_OFF_IN + ST_IN_H * ST_IN_LD * 4;
constexpr int ST_SMEM = ST_OFF_BAR + 64 + 1024;
constexpr int ST_NLD = (ST_IN_H * ST_IN_W + ST_THREADS - 1) / ST_THREADS;  // window floats per thread
static_assert(ST_SMEM <= 227 * 1024, "stem shared memory");
static_assert(ST_PH * ST_PW * 8 <= ST_THREADS, "one thread per (pooled pixel, 8 channels) of a step");

struct alignas(64) StemParams {
    CUtensorMap mapB;                     // weights (192, 64[, 2]) fp16, box (64, 64[, 2])
    int nimg, pool;
    int unit_start[RF_MAX_IMGS + 1];      // prefix sums of steps per image; [nimg ..] = all steps
    int steps[RF_MAX_IMGS];               // steps per strip
    int H[RF_MAX_IMGS], W[RF_MAX_IMGS];   // input image
    int Hs[RF_MAX_IMGS], Ws[RF_MAX_IMGS]; // stem output
    int Ho[RF_MAX_IMGS], Wo[RF_MAX_IMGS]; // stored output: pooled (pool = 1) or the stem output
    long long in_pix[RF_MAX_IMGS], out_pix[RF_MAX_IMGS];
    long long plane;                      // split output: elements from the hi to the lo plane
    const float* x;
    const float* bias;
    __half* y;
};

// one staged window element: (hi, lo * 2^11) fp16 pair packed in 32 bits (hi in the low half)
__device__ __forceinline__ uint32_t stem_pack_split(float v) {
    __half2 hi, lo;
    split2(v, 0.f, hi, lo);
    return (*reinterpret_cast<uint32_t*>(&hi) & 0xFFFFu) | (*reinterpret_cast<uint32_t*>(&lo) << 16);
}

// half a patch: the 16-byte chunks 4 * HALF .. 4 * HALF + 3 of K block kb of pixel m, hi (and lo) planes
template <bool SPLIT, int HALF, int kb>
__device__ __forceinline__ void stem_build_half(const uint32_t* __restrict__ base, uint8_t* sA, int m) {
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
        const int c8 = HALF * 4 + cc;
        uint4 oh, ol;
        uint32_t* ph = reinterpret_cast<uint32_t*>(&oh);
        uint32_t* pl = reinterpret_cast<uint32_t*>(&ol);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k0 = kb * 64 + c8 * 8 + 2 * e, k1 = k0 + 1;
            const uint32_t a = k0 < ST_KK ? base[(k0 / 21) * ST_IN_LD + (k0 % 21)] : 0u;
            const uint32_t b = k1 < ST_KK ? base[(k1 / 21) * ST_IN_LD + (k1 % 21)] : 0u;
            ph[e] = __byte_perm(a, b, 0x5410);          // (hi(a), hi(b))
            pl[e] = __byte_perm(a, b, 0x7632);          // (lo(a), lo(b))
        }
        uint8_t* dst = sA + kb * TC_A_BYTES + m * 128 + ((c8 ^ (m & 7)) << 4);
        *reinterpret_cast<uint4*>(dst) = oh;
        if constexpr (SPLIT) *reinterpret_cast<uint4*>(dst + ST_OFF_ALO) = ol;
    }
}

// K block kb of a step: build it, hand it to the async proxy, issue its wgmmas (one commit group)
template <bool SPLIT, int kb, int NACC>
__device__ __forceinline__ void stem_kblock(float (&acc)[NACC][32], const uint32_t* base, uint8_t* sA, const uint8_t* sB, int m, int half,
                                            int g, uint64_t* bar_b, bool first) {
    constexpr int NPL = SPLIT ? 2 : 1;
    if (half == 0) stem_build_half<SPLIT, 0, kb>(base, sA, m);
    else stem_build_half<SPLIT, 1, kb>(base, sA, m);
    fence_proxy_async();            // generic-proxy writes -> visible to the tensor core (async proxy)
    __syncthreads();
    if (kb == 0 && first) mbar_wait(bar_b, 0);
    wg_fence();
    const uint32_t a = smem_u32(sA + kb * TC_A_BYTES + g * (64 * 128)), b = smem_u32(sB + kb * NPL * ST_B_PLANE);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t ah = wg_desc(a + 32 * k), bh = wg_desc(b + 32 * k);
        if constexpr (SPLIT) {
            wgmma<false, 64>(acc[1], wg_desc(a + ST_OFF_ALO + 32 * k), bh);
            wgmma<false, 64>(acc[1], ah, wg_desc(b + ST_B_PLANE + 32 * k));
        }
        wgmma<false, 64>(acc[0], ah, bh);
    }
    wg_commit();
}

template <bool SPLIT>
__global__ void __launch_bounds__(ST_THREADS, 1)
stem7_kernel(const __grid_constant__ StemParams p) {
    constexpr int NPL = SPLIT ? 2 : 1;
    constexpr int NACC = SPLIT ? 2 : 1;
    constexpr int PIX_BYTES = SPLIT ? 256 : 128;    // one stem pixel in a shared tile: 64 fp32 (engine 2: fp16)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + ST_OFF_B;
    uint8_t* sT = smem + ST_OFF_T;
    uint32_t* sIn = reinterpret_cast<uint32_t*>(smem + ST_OFF_IN);
    uint64_t* bar_b = reinterpret_cast<uint64_t*>(smem + ST_OFF_BAR);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31, g = warp >> 2;
    const long long units = p.unit_start[RF_MAX_IMGS];
    const int u_begin = (int)(units * blockIdx.x / gridDim.x), u_end = (int)(units * (blockIdx.x + 1) / gridDim.x);

    struct Unit { int img, strip, j, r0, c0; };
    auto decode = [&](int u) {
        Unit U;
        U.img = 0;
#pragma unroll
        for (int i = 1; i < RF_MAX_IMGS; ++i) U.img += (i < p.nimg && u >= p.unit_start[i]) ? 1 : 0;
        const int loc = u - p.unit_start[U.img];
        U.strip = loc / p.steps[U.img];
        U.j = loc - U.strip * p.steps[U.img];
        U.r0 = U.j * ST_TH;
        U.c0 = p.pool ? U.strip * 2 * ST_PW - 1 : U.strip * ST_TW;
        return U;
    };
    float win[ST_NLD];
    auto load_window = [&](const Unit& U) {         // the zero-padded input window of a step, into registers
        const int H = p.H[U.img], WC = p.W[U.img] * ST_C;
        const float* src = p.x + p.in_pix[U.img] * ST_C;
        const int iy0 = U.r0 * 2 - 3, col0 = (U.c0 * 2 - 3) * ST_C;
#pragma unroll
        for (int i = 0; i < ST_NLD; ++i) {
            const int idx = t + i * ST_THREADS;
            const int r = idx / ST_IN_W, jj = idx - r * ST_IN_W;
            const int iy = iy0 + r, col = col0 + jj;
            win[i] = (idx < ST_IN_H * ST_IN_W && iy >= 0 && iy < H && col >= 0 && col < WC) ? __ldg(src + (long long)iy * WC + col) : 0.f;
        }
    };
    auto stage_window = [&]() {                     // ... split once, into shared memory
#pragma unroll
        for (int i = 0; i < ST_NLD; ++i) {
            const int idx = t + i * ST_THREADS;
            const int r = idx / ST_IN_W, jj = idx - r * ST_IN_W;
            if (idx < ST_IN_H * ST_IN_W) sIn[r * ST_IN_LD + jj] = stem_pack_split(win[i]);
        }
    };

    if (t == 0) {
        mbar_init(bar_b, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (t == 0) {
        mbar_expect_tx(bar_b, ST_KB * NPL * ST_B_PLANE);
#pragma unroll
        for (int kb = 0; kb < ST_KB; ++kb) {
            if constexpr (SPLIT) tma_load_3d(sB + kb * 2 * ST_B_PLANE, &p.mapB, bar_b, kb * 64, 0, 0);
            else tma_load_2d(sB + kb * ST_B_PLANE, &p.mapB, bar_b, kb * 64, 0);
        }
    }
    int u = u_begin;
    Unit U = decode(u);
    if (p.pool && U.j > 0) U = decode(--u);         // the step above the range: its last stem row, not pooled
    load_window(U);
    stage_window();
    __syncthreads();

    // this thread's pixel and patch half: element k = r*21 + s*3 + c of pixel (py, px) sits at sIn[2*py + r][6*px + (k % 21)]
    const int m = t & 127, half = t >> 7;
    const uint32_t* base = sIn + (2 * (m >> 5)) * ST_IN_LD + 6 * (m & 31);
    // accumulator fragment: d[4j + 2h + e] = pixel rbase + 8h, channel 8j + cbase + e
    const int rbase = 64 * g + 16 * (warp & 3) + (lane >> 2), cbase = 2 * (lane & 3);
    int buf = 0;
    for (bool first = true; u < u_end; ++u, first = false) {
        float acc[NACC][32];
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[a][i] = 0.f;
        stem_kblock<SPLIT, 0>(acc, base, sA, sB, m, half, g, bar_b, first);
        stem_kblock<SPLIT, 1>(acc, base, sA, sB, m, half, g, bar_b, first);
        stem_kblock<SPLIT, 2>(acc, base, sA, sB, m, half, g, bar_b, first);
        const bool more = u + 1 < u_end;
        Unit N = U;
        if (more) {
            N = decode(u + 1);
            load_window(N);
        }
        wg_wait<0>();
#pragma unroll
        for (int a = 0; a < NACC; ++a) wg_fence_regs(acc[a]);

        const int img = U.img;
        uint8_t* tile = sT + buf * ST_T_BYTES;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int mm = rbase + 8 * h;
            const int oy = U.r0 + (mm >> 5), ox = U.c0 + (mm & 31);
            __half* y = p.y + (p.out_pix[img] + (long long)oy * p.Wo[img] + ox) * 64;
            const bool store = !p.pool && oy < p.Hs[img] && ox < p.Ws[img];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = 8 * j + cbase, i = 4 * j + 2 * h;
                float v0 = SPLIT ? fmaf(acc[NACC - 1][i], 0.00048828125f, acc[0][i]) : acc[0][i];
                float v1 = SPLIT ? fmaf(acc[NACC - 1][i + 1], 0.00048828125f, acc[0][i + 1]) : acc[0][i + 1];
                if (p.bias) { v0 += __ldg(p.bias + n); v1 += __ldg(p.bias + n + 1); }
                v0 = fmaxf(v0, 0.f);
                v1 = fmaxf(v1, 0.f);
                if constexpr (SPLIT) {
                    __half2 hi, lo;
                    split2(v0, v1, hi, lo);
                    if (p.pool) {                   // rebuilt as the max-pool of a split tensor reads it
                        const float2 fh = __half22float2(hi), fl = __half22float2(lo);
                        *reinterpret_cast<float2*>(tile + mm * PIX_BYTES + (((n >> 2) ^ (mm & 7)) << 4) + (n & 3) * 4) =
                            make_float2(fmaf(fl.x, 0.00048828125f, fh.x), fmaf(fl.y, 0.00048828125f, fh.y));
                    } else if (store) {
                        *reinterpret_cast<__half2*>(y + n) = hi;
                        *reinterpret_cast<__half2*>(y + p.plane + n) = lo;
                    }
                } else {
                    if (p.pool) *reinterpret_cast<__half2*>(tile + mm * PIX_BYTES + ((j ^ (mm & 7)) << 4) + cbase * 2) = pack_sat(v0, v1);
                    else if (store) *reinterpret_cast<__half2*>(y + n) = pack_sat(v0, v1);
                }
            }
        }
        if (more) stage_window();
        __syncthreads();

        if (p.pool && u >= u_begin && t < ST_PH * ST_PW * 8) {
            // pooled pixel (oy, ox), channels 8 oct .. 8 oct + 7: stem rows 2 oy - 1 .. 2 oy + 1 are tile rows 2 pr - 1 .. 2 pr + 1
            // (row -1: the previous step's last row, in the other tile), stem columns 2 ox - 1 .. 2 ox + 1 are tile columns 2 pc ..
            const int oct = t & 7, q = t >> 3, pr = q / ST_PW, pc = q - pr * ST_PW;
            const int oy = U.j * ST_PH + pr, ox = U.strip * ST_PW + pc;
            if (oy < p.Ho[img] && ox < p.Wo[img]) {
                float mx[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) mx[e] = -INFINITY;
                const __half2 ninf = __float2half2_rn(-INFINITY);
                __half2 mh[4] = {ninf, ninf, ninf, ninf};
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const int tr = 2 * pr - 1 + r;
                    if (U.r0 + tr < 0 || U.r0 + tr >= p.Hs[img]) continue;
                    const uint8_t* trow = tr < 0 ? sT + (buf ^ 1) * ST_T_BYTES + 3 * 32 * PIX_BYTES : tile + tr * 32 * PIX_BYTES;
#pragma unroll
                    for (int s = 0; s < 3; ++s) {
                        const int tc = 2 * pc + s;
                        if (U.c0 + tc < 0 || U.c0 + tc >= p.Ws[img]) continue;
                        const uint8_t* px = trow + tc * PIX_BYTES;
                        if constexpr (SPLIT) {
                            const float4 a = *reinterpret_cast<const float4*>(px + (((2 * oct) ^ (tc & 7)) << 4));
                            const float4 b = *reinterpret_cast<const float4*>(px + (((2 * oct + 1) ^ (tc & 7)) << 4));
                            mx[0] = fmaxf(mx[0], a.x); mx[1] = fmaxf(mx[1], a.y); mx[2] = fmaxf(mx[2], a.z); mx[3] = fmaxf(mx[3], a.w);
                            mx[4] = fmaxf(mx[4], b.x); mx[5] = fmaxf(mx[5], b.y); mx[6] = fmaxf(mx[6], b.z); mx[7] = fmaxf(mx[7], b.w);
                        } else {
                            const uint4 v = *reinterpret_cast<const uint4*>(px + ((oct ^ (tc & 7)) << 4));
                            const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                            for (int e = 0; e < 4; ++e) mh[e] = __hmax2(mh[e], hv[e]);
                        }
                    }
                }
                __half* y = p.y + (p.out_pix[img] + (long long)oy * p.Wo[img] + ox) * 64 + oct * 8;
                if constexpr (SPLIT) {
                    split_store8(y, p.plane, mx);
                } else {
                    uint4 o;
                    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
                    for (int e = 0; e < 4; ++e) ho[e] = mh[e];
                    *reinterpret_cast<uint4*>(y) = o;
                }
            }
        }
        buf ^= 1;
        U = N;
    }
}

// hi = x with the 13 low mantissa bits cleared (exactly representable in TF32), lo = x - hi (exact in fp32)
__global__ void split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo, long long n4) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 v = __ldg(x + i), h, l;
    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); l.x = v.x - h.x;
    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u); l.y = v.y - h.y;
    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); l.z = v.z - h.z;
    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u); l.w = v.w - h.w;
    hi[i] = h;
    lo[i] = l;
}

// fp16 split for the correlation (precision 2): hi = fp16(x), lo = fp16((x - hi) * 2^11), both feature matrices in ONE
// launch (hi/lo of A then hi/lo of B are consecutive in the workspace), and the arg-max keys zeroed by the first threads:
// replaces a memset node and two split launches.
__global__ void split_f16_all_kernel(const float4* __restrict__ A, const float4* __restrict__ B, uint2* __restrict__ Ahi, uint2* __restrict__ Alo,
                                     uint2* __restrict__ Bhi, uint2* __restrict__ Blo, long long na4, long long nb4,
                                     unsigned long long* __restrict__ keys, long long nkeys) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nkeys) keys[i] = 0ull;
    if (i >= na4 + nb4) return;
    const bool isA = i < na4;
    const long long k = isA ? i : i - na4;
    const float4 v = __ldg((isA ? A : B) + k);
    const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    const __half2 l0 = __floats2half2_rn((v.x - f0.x) * 2048.f, (v.y - f0.y) * 2048.f);
    const __half2 l1 = __floats2half2_rn((v.z - f1.x) * 2048.f, (v.w - f1.y) * 2048.f);
    uint2 ho, lo2;
    ho.x = *reinterpret_cast<const uint32_t*>(&h0); ho.y = *reinterpret_cast<const uint32_t*>(&h1);
    lo2.x = *reinterpret_cast<const uint32_t*>(&l0); lo2.y = *reinterpret_cast<const uint32_t*>(&l1);
    (isA ? Ahi : Bhi)[k] = ho;
    (isA ? Alo : Blo)[k] = lo2;
}

// ------------------------------------------------------------------ host side: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

struct MapKey {
    const void* ptr;
    unsigned long long d0, d1, d2, d3, plane;
    unsigned b0, b1, b2, b3, es, esize;
    bool operator==(const MapKey& o) const {
        return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 && plane == o.plane && b0 == o.b0 && b1 == o.b1 && b2 == o.b2 &&
               b3 == o.b3 && es == o.es && esize == o.esize;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = std::hash<const void*>()(k.ptr);
        auto mix = [&](unsigned long long v) { h ^= std::hash<unsigned long long>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.d0); mix(k.d1); mix(k.d2); mix(k.d3); mix(k.plane); mix(k.b0); mix(k.b1); mix(k.b2); mix(k.b3); mix(k.es); mix(k.esize);
        return h;
    }
};
static std::mutex g_map_mu;
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// fp32 (esize 4) or fp16 (esize 2) tensor (d0 innermost, d1, d2[, d3]), dense strides (the 4-D form: d3 planes `plane_bytes`
// apart), box of (b0, b1, b2[, b3]) ELEMENTS LOADED, traversal stride `es` on d1 / d2 (strided convolutions: every es-th
// pixel), 128B swizzle, zero fill out of bounds
int get_map4(CUtensorMap* out, const void* ptr, unsigned long long d0, unsigned long long d1, unsigned long long d2, unsigned long long d3,
             unsigned long long plane_bytes, unsigned b0, unsigned b1, unsigned b2, unsigned b3, unsigned es_, unsigned esize) {
    MapKey key{ptr, d0, d1, d2, d3, plane_bytes, b0, b1, b2, b3, es_, esize};
    std::lock_guard<std::mutex> g(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return 0; }
    EncodeTiledFn enc = get_encode();
    if (!enc) return fail_msg("cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[4] = {d0, d1, d2, d3};
    cuuint64_t strides[3] = {d0 * (unsigned long long)esize, d0 * d1 * (unsigned long long)esize, plane_bytes};
    cuuint32_t box[4] = {b0, b1 * es_, b2 * es_, b3};      // bounding box in tensor coordinates; ceil(box / stride) elements are loaded
    cuuint32_t es[4] = {1, es_, es_, 1};
    int rank = d3 > 0 ? 4 : (d2 > 0 ? 3 : 2);
    CUresult r = enc(out, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(ptr), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(g_err, sizeof(g_err), "cuTensorMapEncodeTiled failed with CUresult %d (dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", (int)r, d0, d1, d2, d3, b0, b1, b2, b3);
        return 3;
    }
    if (g_maps.size() > 8192) g_maps.clear();
    g_maps[key] = *out;
    return 0;
}

int get_map(CUtensorMap* out, const void* ptr, unsigned long long d0, unsigned long long d1, unsigned long long d2,
            unsigned b0, unsigned b1, unsigned b2, unsigned es_, unsigned esize) {
    return get_map4(out, ptr, d0, d1, d2, 0, 0, b0, b1, b2, 0, es_, esize);
}

int pick_tw(int Ho, int Wo) {
    // tile = tw x (128/tw) output pixels: minimise the padded area
    int best = 16;
    long long best_area = -1;
    const int cands[5] = {16, 32, 8, 64, 128};
    for (int i = 0; i < 5; ++i) {
        int tw = cands[i], th = 128 / tw;
        long long area = (long long)((Wo + tw - 1) / tw) * ((Ho + th - 1) / th);
        if (best_area < 0 || area < best_area) { best_area = area; best = tw; }
    }
    return best;
}

template <int KIND, int BN, int MODE, int OUT>
static int launch_wg(const WgParams& p, dim3 grid, cudaStream_t st) {
    using Cfg = WgCfg<KIND, BN, MODE>;
    static bool attr[64] = {false};
    const int dev = current_device();
    if (!attr[dev]) {
        RF_CUDA(cudaFuncSetAttribute(wg_kernel<KIND, BN, MODE, OUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr[dev] = true;
    }
    wg_kernel<KIND, BN, MODE, OUT><<<grid, WG_THREADS, Cfg::SMEM_BYTES, st>>>(p);
    RF_LAUNCHED();
    return 0;
}

// persistent: at most as many CTAs as fit the GPU at once, each looping over its share of the tiles
template <int KIND, int BN, int OUT>
static int launch_conv_bn(const WgParams& p, cudaStream_t st) {
    const int resident = WgCfg<KIND, BN, MODE_CONV>::CTAS_PER_SM * num_sms();
    return launch_wg<KIND, BN, MODE_CONV, OUT>(p, dim3(p.ntiles < resident ? p.ntiles : resident), st);
}
template <int KIND, int OUT>
static int launch_conv(const WgParams& p, int BN, cudaStream_t st) {
    return BN == 128 ? launch_conv_bn<KIND, 128, OUT>(p, st) : launch_conv_bn<KIND, 64, OUT>(p, st);
}

// dual: a second input (x2, its own per-image sizes hw2, Cin2 channels, sampled with stride2) whose channels continue the K axis
// of a 1x1 convolution: y = act(W[:, :Cin] x + W[:, Cin:] x2[::stride2] + bias) - a bottleneck's conv3 and its down-sampling
// branch in one GEMM (the branch's output never goes to HBM and comes back as a residual).
struct SplitDual { const void* x2; const int* hw2; int Cin2, stride2; };

// kind K_TF32: x / residual / y fp32, w [Cout][K] fp32.  K_F16: fp16 x / residual / w, y fp16 (out32: fp32).  K_SPLIT: x / residual /
// y split tensors ([2][P][C] fp16, planes P * C elements apart), w [2][Cout][K] fp16 (out32: y fp32 [P][Cout], no residual).
static int conv_impl(const ImgSet& batch, const ConvParams& cp, const void* w, cudaStream_t st, int kind, bool out32, const SplitDual* dual) {
    // Flat tiles: the pixels of a 1x1 / stride-1 layer are independent rows of the batch's [sum HW][C] matrix (its second input's
    // too, at stride2 = 1), so the batch runs as ONE image of 1 x sum(HW) pixels, in tiles of 128 consecutive pixels that run on
    // across image boundaries.  Only the batch's last tile is partial; the tensor maps' bounds clip it.  3x3 and strided layers
    // keep per-image tw x (128 / tw) tiles, the shape their halo and traversal stride need.
    const bool flat = cp.R == 1 && cp.S == 1 && cp.stride == 1 && cp.pad == 0 && (dual == nullptr || dual->stride2 == 1);
    int hw_flat[2] = {1, 0};
    ImgSet flat_set;
    if (flat) {
        RF_REQUIRE(batch.out_pix[batch.n] <= INT_MAX, "rf_conv2d_nhwc: more than 2^31 - 1 pixels in one batch");
        hw_flat[1] = (int)batch.out_pix[batch.n];
        RF_REQUIRE(make_imgset(flat_set, 1, hw_flat, 1, 1, 0) == 0, "rf_conv2d_nhwc: bad image set");
    }
    const ImgSet& set = flat ? flat_set : batch;
    const int* hw2 = dual == nullptr ? nullptr : flat ? hw_flat : dual->hw2;
    WgParams p;
    memset(&p, 0, sizeof(p));
    const bool split = kind == K_SPLIT;
    const unsigned esz = kind == K_TF32 ? 4u : 2u;
    const unsigned bk = kind == K_TF32 ? TC_BK : TC_BK_F16;
    const int BN = cp.Cout > 64 ? 128 : 64;
    const char* xb = reinterpret_cast<const char*>(cp.x);
    const unsigned long long in_plane = (unsigned long long)set.in_pix[set.n] * cp.Cin * 2ull;
    long long in2_pix[RF_MAX_IMGS + 1] = {0};
    if (dual)
        for (int i = 0; i < set.n; ++i) in2_pix[i + 1] = in2_pix[i] + (long long)hw2[2 * i] * hw2[2 * i + 1];
    const unsigned long long in2_plane = dual ? (unsigned long long)in2_pix[set.n] * dual->Cin2 * 2ull : 0ull;
    p.nimg = set.n;
    const bool tma_out = kind != K_TF32 && !out32;          // fp16 / split outputs: stored (and their residual loaded) by TMA
    const unsigned long long out_plane = (unsigned long long)set.out_pix[set.n] * cp.Cout * 2ull;
    const char* yb = reinterpret_cast<const char*>(cp.y);
    const char* rb = reinterpret_cast<const char*>(cp.residual);
    int tiles = 0;
    for (int i = 0; i < set.n; ++i) {
        const int tw = flat ? 128 : pick_tw(set.Ho[i], set.Wo[i]), th = 128 / tw;
        p.tw[i] = tw;
        p.tiles_x[i] = (set.Wo[i] + tw - 1) / tw;
        p.tile_start[i] = tiles;
        tiles += p.tiles_x[i] * ((set.Ho[i] + th - 1) / th);
        p.Ho[i] = set.Ho[i]; p.Wo[i] = set.Wo[i];
        p.out_pix[i] = set.out_pix[i];
        int rc = split ? get_map4(&p.mapA[i], xb + set.in_pix[i] * cp.Cin * 2, (unsigned long long)cp.Cin, (unsigned long long)set.W[i],
                                  (unsigned long long)set.H[i], 2, in_plane, bk, (unsigned)tw, (unsigned)th, 2, (unsigned)cp.stride, 2)
                       : get_map(&p.mapA[i], xb + set.in_pix[i] * cp.Cin * esz, (unsigned long long)cp.Cin, (unsigned long long)set.W[i],
                                 (unsigned long long)set.H[i], bk, (unsigned)tw, (unsigned)th, (unsigned)cp.stride, esz);
        if (!rc && dual)
            rc = get_map4(&p.mapA2[i], static_cast<const char*>(dual->x2) + in2_pix[i] * dual->Cin2 * 2, (unsigned long long)dual->Cin2,
                          (unsigned long long)hw2[2 * i + 1], (unsigned long long)hw2[2 * i], 2, in2_plane, bk, (unsigned)tw,
                          (unsigned)th, 2, (unsigned)dual->stride2, 2);
        // output and residual maps: the image's own pixels and the layer's Cout channels, so that the bounds clip partial tiles
        const long long o = set.out_pix[i] * cp.Cout * 2;
        for (int m = 0; m < (cp.residual ? 2 : 1) && tma_out && !rc; ++m) {
            CUtensorMap* map = m == 0 ? &p.mapY[i] : &p.mapR[i];
            const void* base = (m == 0 ? yb : rb) + o;
            rc = split ? get_map4(map, base, (unsigned long long)cp.Cout, (unsigned long long)set.Wo[i], (unsigned long long)set.Ho[i], 2,
                                  out_plane, 64, (unsigned)tw, (unsigned)th, 2, 1, 2)
                       : get_map(map, base, (unsigned long long)cp.Cout, (unsigned long long)set.Wo[i], (unsigned long long)set.Ho[i],
                                 64, (unsigned)tw, (unsigned)th, 1, 2);
        }
        if (rc) return rc;
    }
    RF_REQUIRE(tiles > 0, "rf_conv2d_nhwc: empty output");
    for (int i = set.n; i <= RF_MAX_IMGS; ++i) p.tile_start[i] = tiles;
    p.out_pix[set.n] = set.out_pix[set.n];
    int rc = split ? get_map(&p.mapB, w, (unsigned long long)cp.K, (unsigned long long)cp.Cout, 2, bk, (unsigned)BN, 2, 1, 2)
                   : get_map(&p.mapB, w, (unsigned long long)cp.K, (unsigned long long)cp.Cout, 0, bk, (unsigned)BN, 0, 1, esz);
    if (rc) return rc;
    p.R = cp.R; p.S = cp.S; p.pad = cp.pad; p.stride = cp.stride; p.Cin = cp.Cin; p.Cout = cp.Cout; p.relu = cp.relu; p.round_out = cp.round_out;
    p.dil = cp.dil;
    p.kc1 = cp.Cin / (int)bk;
    p.stride2 = 1;
    if (dual) { p.Cin = cp.Cin + dual->Cin2; p.stride2 = dual->stride2; }      // the kernel's K axis: both inputs
    p.plane = (long long)set.out_pix[set.n] * cp.Cout;
    p.bias = cp.bias; p.residual = cp.residual; p.y = cp.y;
    p.ntiles = tiles * ((cp.Cout + BN - 1) / BN);
    if (kind == K_TF32) return launch_conv<K_TF32, O_F32>(p, BN, st);
    if (kind == K_F16) return out32 ? launch_conv<K_F16, O_F32>(p, BN, st) : launch_conv<K_F16, O_F16>(p, BN, st);
    return out32 ? launch_conv<K_SPLIT, O_F32>(p, BN, st) : launch_conv<K_SPLIT, O_SPLIT>(p, BN, st);
}

template <bool SPLIT>
static int stem_impl(const float* x, int nimg, const int* hw_host, const void* w, const float* bias, void* y, int pool, void* stream) {
    RF_REQUIRE(x != nullptr && w != nullptr && y != nullptr, "rf_stem7: null pointer");
    RF_REQUIRE(((uintptr_t)y % 16) == 0 && ((uintptr_t)w % 16) == 0, "rf_stem7: pointers must be 16-byte aligned");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw_host, 7, 2, 3) == 0, "rf_stem7: bad image set");
    StemParams p;
    memset(&p, 0, sizeof(p));
    p.nimg = nimg;
    p.pool = pool ? 1 : 0;
    int units = 0;
    long long out = 0;
    for (int i = 0; i < nimg; ++i) {
        const int Hs = set.Ho[i], Ws = set.Wo[i];
        const int Ho = pool ? (Hs - 1) / 2 + 1 : Hs, Wo = pool ? (Ws - 1) / 2 + 1 : Ws;      // max-pool 3 / stride 2 / pad 1
        const int strips = pool ? (Wo + ST_PW - 1) / ST_PW : (Ws + ST_TW - 1) / ST_TW;
        p.steps[i] = pool ? (Ho + ST_PH - 1) / ST_PH : (Hs + ST_TH - 1) / ST_TH;
        p.unit_start[i] = units;
        units += strips * p.steps[i];
        p.H[i] = set.H[i]; p.W[i] = set.W[i]; p.Hs[i] = Hs; p.Ws[i] = Ws; p.Ho[i] = Ho; p.Wo[i] = Wo;
        p.in_pix[i] = set.in_pix[i];
        p.out_pix[i] = out;
        out += (long long)Ho * Wo;
    }
    for (int i = nimg; i <= RF_MAX_IMGS; ++i) p.unit_start[i] = units;
    int rc = SPLIT ? get_map(&p.mapB, w, 192ull, 64ull, 2, 64, 64, 2, 1, 2) : get_map(&p.mapB, w, 192ull, 64ull, 0, 64, 64, 0, 1, 2);
    if (rc) return rc;
    p.plane = out * 64;
    p.x = x; p.bias = bias; p.y = static_cast<__half*>(y);
    static bool attr[64] = {false};
    const int dev = current_device();
    if (!attr[dev]) {
        RF_CUDA(cudaFuncSetAttribute(stem7_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_SMEM));
        attr[dev] = true;
    }
    const int grid = units < num_sms() ? units : num_sms();
    stem7_kernel<SPLIT><<<grid, ST_THREADS, ST_SMEM, as_stream(stream)>>>(p);
    RF_LAUNCHED();
    return 0;
}

}  // namespace rf

using namespace rf;

bool rf_conv2d_tc_supported(const ConvParams& p) {
    return (p.stride == 1 || p.stride == 2) && (p.Cin % TC_BK) == 0 && p.Cout >= 1 && p.R == p.S && (p.R == 1 || p.R == 3);
}
// engine 2: fp16 activations / weights; every layer must fit (there is no fp16 SIMT path to fall back to)
bool rf_conv2d_f16_supported(const ConvParams& p) {
    return (p.stride == 1 || p.stride == 2) && (p.Cin % TC_BK_F16) == 0 && p.Cout >= 8 && (p.Cout % 8) == 0 && p.R == p.S && (p.R == 1 || p.R == 3);
}
bool rf_conv2d_split_supported(const ConvParams& p) {
    return (p.stride == 1 || p.stride == 2) && (p.Cin % TC_BK_F16) == 0 && p.Cout >= 1 && p.R == p.S && (p.R == 1 || p.R == 3);
}

// f16 = false: x / residual / y fp32, w_tc fp32 [Cout][K] (TF32-rounded).  f16 = true: the same pointers hold IEEE fp16.
// out32 (with f16): y is fp32 (3x3 / stride 1 layers only, no residual) - the hand-over from fp16 layers to a TF32 consumer.
int rf_conv2d_tc(const ImgSet& set, const ConvParams& cp, const void* w_tc, cudaStream_t st, bool f16, bool out32) {
    RF_REQUIRE(w_tc != nullptr, "rf_conv2d_nhwc: tensor-core engines need w_tc ([Cout][R*S*Cin])");
    RF_REQUIRE(f16 ? rf_conv2d_f16_supported(cp) : rf_conv2d_tc_supported(cp),
               "rf_conv2d_nhwc: tensor-core engines need stride 1 or 2, 1x1 or 3x3, Cin % 32 == 0 (fp16: Cin % 64 == 0, Cout % 8 == 0)");
    RF_REQUIRE(!out32 || (f16 && cp.R == 3 && cp.stride == 1 && cp.pad == 1 && cp.residual == nullptr),
               "rf_conv2d_nhwc: engine 3 (fp16 operands, fp32 output) covers 3x3 / stride 1 / pad 1 layers without residual");
    RF_REQUIRE(!f16 || (((uintptr_t)cp.x % 16) == 0 && ((uintptr_t)cp.y % 16) == 0 && ((uintptr_t)cp.residual % 16) == 0),
               "rf_conv2d_nhwc: engine 2 needs 16-byte aligned x / y / residual");
    return conv_impl(set, cp, w_tc, st, f16 ? K_F16 : K_TF32, out32, nullptr);
}

int rf_conv2d_split(const ImgSet& set, const ConvParams& cp, const void* w_split, cudaStream_t st, bool out32) {
    RF_REQUIRE(w_split != nullptr, "rf_conv2d_nhwc: engine 4 needs the split weights ([2][Cout][R*S*Cin] fp16)");
    RF_REQUIRE(rf_conv2d_split_supported(cp), "rf_conv2d_nhwc: engine 4 needs stride 1 or 2, 1x1 or 3x3, Cin % 64 == 0");
    RF_REQUIRE(out32 || (cp.Cout % 8) == 0, "rf_conv2d_nhwc: engine 4 needs Cout % 8 == 0 for split outputs");
    RF_REQUIRE(!out32 || cp.residual == nullptr, "rf_conv2d_nhwc: engine 4 fp32 outputs take no residual");
    RF_REQUIRE(cp.dil == 1 || (!out32 && cp.R == 3 && cp.stride == 1), "rf_conv2d_nhwc: dilation needs engine 4, a 3x3 kernel and stride 1");
    RF_REQUIRE(((uintptr_t)cp.x % 16) == 0 && ((uintptr_t)cp.y % 16) == 0 && ((uintptr_t)cp.residual % 16) == 0 && ((uintptr_t)w_split % 16) == 0,
               "rf_conv2d_nhwc: engine 4 needs 16-byte aligned pointers");
    return conv_impl(set, cp, w_split, st, K_SPLIT, out32, nullptr);
}

extern "C" int rf_conv1x1_dual_split(const void* x1, const void* x2, int nimg, const int* hw1_host, const int* hw2_host, int Cin1, int Cin2,
                                     int stride2, const void* w_split, const float* bias, int Cout, int relu, void* y, void* stream) {
    RF_REQUIRE(x1 != nullptr && x2 != nullptr && y != nullptr && hw1_host != nullptr && hw2_host != nullptr && w_split != nullptr,
               "rf_conv1x1_dual_split: null pointer");
    RF_REQUIRE(Cin1 >= 1 && Cin2 >= 1 && Cout >= 1, "rf_conv1x1_dual_split: bad channel counts");
    RF_REQUIRE((Cin1 % TC_BK_F16) == 0 && (Cin2 % TC_BK_F16) == 0 && (Cout % 8) == 0 && (stride2 == 1 || stride2 == 2),
               "rf_conv1x1_dual_split: Cin1 % 64 == 0, Cin2 % 64 == 0, Cout % 8 == 0, stride2 1 or 2");
    RF_REQUIRE(((uintptr_t)x1 % 16) == 0 && ((uintptr_t)x2 % 16) == 0 && ((uintptr_t)y % 16) == 0 && ((uintptr_t)w_split % 16) == 0,
               "rf_conv1x1_dual_split: pointers must be 16-byte aligned");
    ImgSet set;
    RF_REQUIRE(make_imgset(set, nimg, hw1_host, 1, 1, 0) == 0, "rf_conv1x1_dual_split: bad image set");
    for (int i = 0; i < nimg; ++i)
        RF_REQUIRE((hw2_host[2 * i] - 1) / stride2 + 1 == set.Ho[i] && (hw2_host[2 * i + 1] - 1) / stride2 + 1 == set.Wo[i],
                   "rf_conv1x1_dual_split: the second input, sampled with stride2, must have the first input's size");
    ConvParams p;
    p.x = static_cast<const float*>(x1); p.w = nullptr; p.bias = bias; p.residual = nullptr; p.y = static_cast<float*>(y);
    p.Cin = Cin1; p.Cout = Cout; p.R = 1; p.S = 1; p.stride = 1; p.pad = 0; p.relu = relu;
    p.round_out = 0;
    p.dil = 1;
    p.Mtot = set.out_pix[nimg];
    p.K = Cin1 + Cin2;
    SplitDual dual{x2, hw2_host, Cin2, stride2};
    return conv_impl(set, p, w_split, as_stream(stream), K_SPLIT, false, &dual);
}

// fused ResNet-50 stem (pool: and its 3x3 / stride 2 / pad 1 max-pool).  x fp32 [sum HW][3], bias fp32 [64]; engine 2: w_f16
// [64][192] ((r, s, c) order, zero padded), y fp16 [sum HoWo][64]; engine 4: w_split [2][64][192], y split [2][sum HoWo][64]
int rf_stem7_f16_impl(const float* x, int nimg, const int* hw_host, const void* w_f16, const float* bias, int pool, void* y_f16, void* stream) {
    return stem_impl<false>(x, nimg, hw_host, w_f16, bias, y_f16, pool, stream);
}
int rf_stem7_split_impl(const float* x, int nimg, const int* hw_host, const void* w_split, const float* bias, int pool, void* y_split, void* stream) {
    return stem_impl<true>(x, nimg, hw_host, w_split, bias, y_split, pool, stream);
}

size_t rf_corr_tc_workspace(int NA, int NB, int C) { return 2ull * ((size_t)NA + NB) * C * sizeof(float) + 1024; }

// Precision 2 splits both operands in one launch that also zeroes rowbest / colbest (contiguous, NA + NB keys); precision 1
// splits them in two launches behind the caller's key memset.
// presplit (precision 2; nullable): {A hi, A lo, B hi, B lo} fp16 planes written by the producer of the features
// (rf_l2norm_split_nhwc): no split launch; the caller has zeroed the keys.
int rf_corr_argmax_tc(const float* featA, int NA, const float* featB, int NB, int C,
                      unsigned long long* rowbest, unsigned long long* colbest, void* ws, cudaStream_t st, int precision,
                      const void* const* presplit) {
    const bool f16 = precision == 2;
    RF_REQUIRE(presplit == nullptr || f16, "rf_corr_mutual_nn: pre-split operands go with the fp16-split kernel (precision 2)");
    RF_REQUIRE((C % (f16 ? TC_BK_F16 : TC_BK)) == 0, "rf_corr_mutual_nn: precision 1 needs C % 32 == 0, precision 2 C % 64 == 0");
    uintptr_t base = (reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255;
    const size_t esz = f16 ? 2 : 4;
    char* Ahi = reinterpret_cast<char*>(base);
    char* Alo = Ahi + (size_t)NA * C * esz;
    char* Bhi = Alo + (size_t)NA * C * esz;
    char* Blo = Bhi + (size_t)NB * C * esz;
    long long na4 = (long long)NA * C / 4, nb4 = (long long)NB * C / 4;
    if (presplit != nullptr) {
        Ahi = const_cast<char*>(static_cast<const char*>(presplit[0]));
        Alo = const_cast<char*>(static_cast<const char*>(presplit[1]));
        Bhi = const_cast<char*>(static_cast<const char*>(presplit[2]));
        Blo = const_cast<char*>(static_cast<const char*>(presplit[3]));
        for (int i = 0; i < 4; ++i) RF_REQUIRE(presplit[i] != nullptr && ((uintptr_t)presplit[i] % 16) == 0, "rf_corr_mutual_nn_presplit: planes must be 16-byte aligned");
    } else if (f16) {
        RF_REQUIRE(colbest == rowbest + NA, "rf_corr_mutual_nn: arg-max keys must be contiguous");
        const long long nkeys = (long long)NA + NB, n = na4 + nb4 > nkeys ? na4 + nb4 : nkeys;
        split_f16_all_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float4*)featA, (const float4*)featB, (uint2*)Ahi, (uint2*)Alo,
                                                                            (uint2*)Bhi, (uint2*)Blo, na4, nb4, rowbest, nkeys);
        RF_LAUNCHED();
    } else {
        split_tf32_kernel<<<(unsigned)((na4 + 255) / 256), 256, 0, st>>>((const float4*)featA, (float4*)Ahi, (float4*)Alo, na4);
        RF_LAUNCHED();
        split_tf32_kernel<<<(unsigned)((nb4 + 255) / 256), 256, 0, st>>>((const float4*)featB, (float4*)Bhi, (float4*)Blo, nb4);
        RF_LAUNCHED();
    }
    constexpr int BN = 128;
    const unsigned bk = f16 ? TC_BK_F16 : TC_BK, es = (unsigned)esz;
    WgParams p;
    memset(&p, 0, sizeof(p));
    p.nimg = 1;
    p.tw[0] = 128;
    p.tiles_x[0] = (NA + 127) / 128;
    for (int i = 1; i <= RF_MAX_IMGS; ++i) p.tile_start[i] = p.tiles_x[0];
    p.Ho[0] = 1; p.Wo[0] = NA;
    int rc = get_map(&p.mapA[0], Ahi, (unsigned long long)C, (unsigned long long)NA, 1, bk, 128, 1, 1, es);
    if (!rc) rc = get_map(&p.mapA2[0], Alo, (unsigned long long)C, (unsigned long long)NA, 1, bk, 128, 1, 1, es);
    if (!rc) rc = get_map(&p.mapB, Bhi, (unsigned long long)C, (unsigned long long)NB, 0, bk, BN, 0, 1, es);
    if (!rc) rc = get_map(&p.mapBlo, Blo, (unsigned long long)C, (unsigned long long)NB, 0, bk, BN, 0, 1, es);
    if (rc) return rc;
    p.R = 1; p.S = 1; p.pad = 0; p.stride = 1; p.Cin = C; p.Cout = NB;
    p.rowbest = rowbest; p.colbest = colbest; p.NA = NA; p.NB = NB;
    const dim3 grid((NB + BN - 1) / BN, p.tiles_x[0]);
    RF_REQUIRE(grid.y <= 65535u, "rf_corr_mutual_nn: NA > 8388480");
    if (f16) return launch_wg<K_SPLIT, BN, MODE_CORR, 0>(p, grid, st);
    return launch_wg<K_TF32X3, BN, MODE_CORR, 0>(p, grid, st);
}
