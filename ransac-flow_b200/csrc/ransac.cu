// Batched RANSAC homography as one persistent kernel (sm_90a).
//
// Replaces utils/outil.py:117-164 (RANSAC), :102-113 (ScoreRANSAC), :68-87
// (Homography: 4-point DLT through numpy/LAPACK SVD) and :97-100 (Prediction).
// The reference drives this from the host in chunks of 100 hypotheses with 16
// D2H copies, a CPU SVD and an H2D copy per chunk; here every hypothesis is
// solved and scored on the device and the chunk semantics (first max inside a
// chunk, strict '>' across chunks, the zero-inlier-chunk early return, the
// unchecked remainder chunk) are reproduced by the last CTA to finish.
//
// DLT null vector: LAPACK dgesdd on an 8x9 matrix returns Vh[8] = (G_1...G_8 e_9)^T
// where G_i are the right Householder reflectors of the unblocked
// lower-bidiagonalisation dgebd2 (sign included); the kernel runs exactly that
// recurrence in fp64, one hypothesis per thread, matrix in registers (fully unrolled).
//
// Scoring uses IEEE fp32 ops in a fixed order without FMA contraction so that
// the inlier masks are bit-identical to oracle/outil_oracle.py.
#include "common.cuh"

namespace rf {

constexpr int RANSAC_THREADS = 256;

struct RansacHeader {
    unsigned long long best_key;   // (gated count << 32) | (0xFFFFFFFF - raw sample index)
    unsigned int ticket;
    int pad;
};

__device__ __forceinline__ double dsign(double a, double b) { return (b >= 0.0) ? fabs(a) : -fabs(a); }

// LAPACK dlapy2: sqrt(x^2 + y^2) without unnecessary overflow
__device__ __forceinline__ double dlapy2(double x, double y) {
    double xa = fabs(x), ya = fabs(y);
    double w = fmax(xa, ya), z = fmin(xa, ya);
    if (z == 0.0) return w;
    double q = z / w;
    return w * sqrt(1.0 + q * q);
}

// 4-point DLT, one hypothesis per thread, the 8x9 fp64 matrix held in REGISTERS (every loop below is fully
// unrolled so all indices are compile-time constants).  Writes the unit-norm null vector (LAPACK's sign) as fp32.
// Same operation order as the dgebd2 recurrence spelled out in oracle/outil_oracle.py::householder_null_vector.
__device__ __forceinline__ void dlt_null_vector(const float (&xu)[4], const float (&xv)[4],
                                                const float (&yu)[4], const float (&yv)[4], float* h_out) {
    double A[8][9];
    // utils/outil.py:73-81: entries are fp32 products upcast to fp64
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float u = yu[i], v = yv[i], u_ = xu[i], v_ = xv[i];
        A[2 * i][0] = 0.0; A[2 * i][1] = 0.0; A[2 * i][2] = 0.0;
        A[2 * i][3] = (double)(-u); A[2 * i][4] = (double)(-v); A[2 * i][5] = -1.0;
        A[2 * i][6] = (double)__fmul_rn(v_, u); A[2 * i][7] = (double)__fmul_rn(v_, v); A[2 * i][8] = (double)v_;
        A[2 * i + 1][0] = (double)u; A[2 * i + 1][1] = (double)v; A[2 * i + 1][2] = 1.0;
        A[2 * i + 1][3] = 0.0; A[2 * i + 1][4] = 0.0; A[2 * i + 1][5] = 0.0;
        A[2 * i + 1][6] = (double)__fmul_rn(-u_, u); A[2 * i + 1][7] = (double)__fmul_rn(-u_, v); A[2 * i + 1][8] = (double)(-u_);
    }
    double taup[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        // ---- dlarfg: right reflector G_i annihilates A(i, i+1:8) ----
        const double alpha = A[i][i];
        double ss = 0.0;
#pragma unroll
        for (int j = i + 1; j < 9; ++j) ss += A[i][j] * A[i][j];
        const double xnorm = sqrt(ss);
        double tau = 0.0;
        if (xnorm != 0.0) {
            const double beta = -dsign(dlapy2(alpha, xnorm), alpha);
            tau = (beta - alpha) / beta;
            const double scal = 1.0 / (alpha - beta);
#pragma unroll
            for (int j = i + 1; j < 9; ++j) A[i][j] *= scal;        // v_i (v_i[i] = 1 implicit)
        }
        taup[i] = tau;
        // ---- dlarf('Right'): rows i+1..7, columns i..8 ----
        if (tau != 0.0) {
#pragma unroll
            for (int r = i + 1; r < 8; ++r) {
                double w = A[r][i];
#pragma unroll
                for (int j = i + 1; j < 9; ++j) w += A[r][j] * A[i][j];
                const double tw = tau * w;
                A[r][i] -= tw;
#pragma unroll
                for (int j = i + 1; j < 9; ++j) A[r][j] -= tw * A[i][j];
            }
        }
        // ---- left reflector H_i annihilates A(i+2:7, i), applied to A(i+1:7, i+1:8) ----
        if (i < 7) {
            const double al = A[i + 1][i];
            double s2 = 0.0;
#pragma unroll
            for (int r = i + 2; r < 8; ++r) s2 += A[r][i] * A[r][i];
            const double xn = sqrt(s2);
            if (xn != 0.0) {
                const double beta = -dsign(dlapy2(al, xn), al);
                const double tauq = (beta - al) / beta;
                const double scal = 1.0 / (al - beta);
#pragma unroll
                for (int r = i + 2; r < 8; ++r) A[r][i] *= scal;    // u (u[i+1] = 1 implicit)
#pragma unroll
                for (int j = i + 1; j < 9; ++j) {
                    double w = A[i + 1][j];
#pragma unroll
                    for (int r = i + 2; r < 8; ++r) w += A[r][i] * A[r][j];
                    const double tw = tauq * w;
                    A[i + 1][j] -= tw;
#pragma unroll
                    for (int r = i + 2; r < 8; ++r) A[r][j] -= tw * A[r][i];
                }
            }
        }
    }
    // h = G_1 G_2 ... G_8 e_9
    double h[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) h[j] = (j == 8) ? 1.0 : 0.0;
#pragma unroll
    for (int i = 7; i >= 0; --i) {
        double d = h[i];
#pragma unroll
        for (int j = i + 1; j < 9; ++j) d += A[i][j] * h[j];
        const double td = taup[i] * d;
        h[i] -= td;
#pragma unroll
        for (int j = i + 1; j < 9; ++j) h[j] -= td * A[i][j];
    }
#pragma unroll
    for (int j = 0; j < 9; ++j) h_out[j] = (float)h[j];
}

// fp32 determinant, partial-pivoting LU, no FMA: same op order as oracle det3().
__device__ __forceinline__ float det3_lu(const float* H) {
    float a[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) a[r][c] = H[r * 3 + c];
    float sign = 1.0f;
    int p = 0;
    float best = fabsf(a[0][0]);
    if (fabsf(a[1][0]) > best) { best = fabsf(a[1][0]); p = 1; }
    if (fabsf(a[2][0]) > best) { best = fabsf(a[2][0]); p = 2; }
    if (p == 1) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { float t = a[0][c]; a[0][c] = a[1][c]; a[1][c] = t; }
        sign = -sign;
    } else if (p == 2) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { float t = a[0][c]; a[0][c] = a[2][c]; a[2][c] = t; }
        sign = -sign;
    }
    if (a[0][0] == 0.0f) return 0.0f;
    float l1 = __fdiv_rn(a[1][0], a[0][0]);
    float l2 = __fdiv_rn(a[2][0], a[0][0]);
    float a11 = __fsub_rn(a[1][1], __fmul_rn(l1, a[0][1]));
    float a12 = __fsub_rn(a[1][2], __fmul_rn(l1, a[0][2]));
    float a21 = __fsub_rn(a[2][1], __fmul_rn(l2, a[0][1]));
    float a22 = __fsub_rn(a[2][2], __fmul_rn(l2, a[0][2]));
    if (fabsf(a21) > fabsf(a11)) {
        float t = a11; a11 = a21; a21 = t;
        t = a12; a12 = a22; a22 = t;
        sign = -sign;
    }
    if (a11 == 0.0f) return 0.0f;
    float l = __fdiv_rn(a21, a11);
    float u22 = __fsub_rn(a22, __fmul_rn(l, a12));
    return __fmul_rn(sign, __fmul_rn(__fmul_rn(a[0][0], a11), u22));
}

// utils/outil.py:97-100 for one match and one H (fixed fp32 op order, no FMA)
__device__ __forceinline__ float reproj_error(const float* H, float x0, float x1, float y0, float y1, float y2) {
    float e0 = __fadd_rn(__fadd_rn(__fmul_rn(y0, H[0]), __fmul_rn(y1, H[1])), __fmul_rn(y2, H[2]));
    float e1 = __fadd_rn(__fadd_rn(__fmul_rn(y0, H[3]), __fmul_rn(y1, H[4])), __fmul_rn(y2, H[5]));
    float e2 = __fadd_rn(__fadd_rn(__fmul_rn(y0, H[6]), __fmul_rn(y1, H[7])), __fmul_rn(y2, H[8]));
    float ex = __fdiv_rn(e0, e2);
    float ey = __fdiv_rn(e1, e2);
    float dx = __fsub_rn(x0, ex);
    float dy = __fsub_rn(x1, ey);
    return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
}

// G hypotheses per group (G in {32, 128}); blockDim = RANSAC_THREADS.
// dynamic smem: float Hs[G][9] | int flags[G]
__global__ void __launch_bounds__(RANSAC_THREADS)
ransac_kernel(const float* __restrict__ match1, const float* __restrict__ match2, int M_host,
              const int* __restrict__ M_dev, const long long* __restrict__ samples, int sample_mode, int nbIter,
              float tol, int chunk, int G,
              RansacHeader* hdr, int* counts, float* Hall, int* chunk_nz,
              float* H_out, long long* nbInlier_out, unsigned char* mask_out, int* status_out,
              const int* __restrict__ slot_in, int* __restrict__ slot_out, int n_tables) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* sH = reinterpret_cast<float*>(smem_raw);
    int* sFlag = reinterpret_cast<int*>(sH + 9 * G);
    __shared__ int s_scan[RANSAC_THREADS / 32];
    __shared__ int s_misc[4];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nwarps = RANSAC_THREADS / 32;
    const int M = (M_dev != nullptr) ? min(*M_dev, M_host) : M_host;
    const int nGroups = (nbIter + G - 1) / G;
    if (slot_in != nullptr) {
        // drawn tables (rf_ransac_homography_drawn): this call reads table *slot_in and passes the next slot on, advanced only
        // when it draws (M >= 4, as the reference returns None before torch.randint otherwise).  slot_out is another buffer
        // than slot_in, so no CTA can read the increment this one writes.
        const int slot = *slot_in;
        samples += (long long)min(slot, n_tables - 1) * nbIter * 4;
        if (blockIdx.x == 0 && threadIdx.x == 0) *slot_out = slot + (M >= 4 ? 1 : 0);
    }

    if (M >= 4) {
        for (int g = blockIdx.x; g < nGroups; g += gridDim.x) {
            // ---- phase A: one thread per hypothesis: dedupe + DLT + det gate ----
            if (tid < G) {
                int i = g * G + tid;
                int flag = -1;                      // -1: no hypothesis / duplicated sample
                if (i < nbIter) {
                    long long s[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        s[k] = samples[(long long)i * 4 + k];
                        // RF_SAMPLES_PHILOX64: the word is (x << 32) | y of curand4(); torch.randint(M) on CUDA returns x % M
                        // for the same generator state (ATen DistributionTemplates.h, range < 2^28): take the high word
                        if (sample_mode == RF_SAMPLES_PHILOX64) s[k] = (long long)((unsigned long long)s[k] >> 32);
                        if (sample_mode != RF_SAMPLES_INDEX) s[k] = s[k] % M;
                    }
                    bool dup = (s[0] == s[1]) | (s[0] == s[2]) | (s[0] == s[3]) | (s[1] == s[2]) | (s[1] == s[3]) | (s[2] == s[3]);
                    bool bad = false;
#pragma unroll
                    for (int k = 0; k < 4; ++k) bad |= (s[k] < 0) | (s[k] >= M);
                    if (!dup && !bad) {
                        float xu[4], xv[4], yu[4], yv[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            xu[k] = match1[s[k] * 3 + 0];
                            xv[k] = match1[s[k] * 3 + 1];
                            yu[k] = match2[s[k] * 3 + 0];
                            yv[k] = match2[s[k] * 3 + 1];
                        }
                        float h[9];
                        dlt_null_vector(xu, xv, yu, yv, h);
#pragma unroll
                        for (int k = 0; k < 9; ++k) { sH[tid * 9 + k] = h[k]; Hall[(long long)i * 9 + k] = h[k]; }
                        float det = det3_lu(h);
                        flag = (det > 1e-6f) ? 1 : 0;       // utils/outil.py:113
                    } else if (!dup && bad) {
                        flag = -1;
                    }
                    if (flag < 0) counts[i] = -1;
                }
                sFlag[tid] = flag;
            }
            __syncthreads();
            // ---- phase B: one warp per hypothesis, lanes over matches ----
            for (int hl = warp; hl < G; hl += nwarps) {
                int flag = sFlag[hl];
                if (flag < 0) continue;
                int i = g * G + hl;
                float H[9];
#pragma unroll
                for (int k = 0; k < 9; ++k) H[k] = sH[hl * 9 + k];
                int cnt = 0;
                if (flag == 1) {
                    for (int m = lane; m < M; m += 32) {
                        float x0 = __ldg(match1 + m * 3), x1 = __ldg(match1 + m * 3 + 1);
                        float y0 = __ldg(match2 + m * 3), y1 = __ldg(match2 + m * 3 + 1), y2 = __ldg(match2 + m * 3 + 2);
                        float err = reproj_error(H, x0, x1, y0, y1, y2);
                        cnt += (err < tol) ? 1 : 0;
                    }
                    cnt = __reduce_add_sync(0xffffffffu, cnt);
                }
                if (lane == 0) {
                    counts[i] = cnt;
                    if (cnt > 0) {
                        unsigned long long key = ((unsigned long long)(unsigned)cnt << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
                        atomicMax(&hdr->best_key, key);
                    }
                }
            }
            __syncthreads();
        }
    }

    // ---- last CTA to finish reproduces the chunk semantics and writes the outputs ----
    __threadfence();
    __syncthreads();
    if (tid == 0) s_misc[0] = (atomicAdd(&hdr->ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (!s_misc[0]) return;
    __threadfence();

    if (M < 4) {
        if (tid == 0) { *status_out = RF_RANSAC_TOO_FEW; *nbInlier_out = 0; }
        for (int k = tid; k < 9; k += blockDim.x) H_out[k] = 0.f;
        for (int m = tid; m < M_host; m += blockDim.x) mask_out[m] = 0;
        return;
    }
    const int nChunksMax = nbIter / chunk + 2;
    for (int c = tid; c < nChunksMax; c += blockDim.x) chunk_nz[c] = 0;
    __syncthreads();
    // order-preserving rank u(i) of every kept hypothesis; per-chunk "any non-zero count"
    int offset = 0;
    for (int base = 0; base < nbIter; base += RANSAC_THREADS) {
        int i = base + tid;
        int c = (i < nbIter) ? __ldcg(counts + i) : -1;
        int keep = (c >= 0) ? 1 : 0;
        int incl = keep;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        int wofs = 0, total = 0;
#pragma unroll
        for (int w = 0; w < RANSAC_THREADS / 32; ++w) {
            int v = s_scan[w];
            if (w < warp) wofs += v;
            total += v;
        }
        if (keep && c > 0) {
            int u = offset + wofs + incl - 1;
            atomicOr(&chunk_nz[u / chunk], 1);
        }
        offset += total;
        __syncthreads();
    }
    const int nU = offset;
    const int nFull = nU / chunk;
    if (tid == 0) s_misc[1] = 0;
    __syncthreads();
    for (int c = tid; c < nFull; c += blockDim.x)
        if (__ldcg(chunk_nz + c) == 0) s_misc[1] = 1;            // utils/outil.py:145-146
    __syncthreads();
    const bool zero_chunk = s_misc[1] != 0;
    const unsigned long long key = *((volatile unsigned long long*)&hdr->best_key);
    int status;
    if (zero_chunk) status = RF_RANSAC_NONE;
    else if (key == 0ull) status = RF_RANSAC_NO_MODEL;  // utils/outil.py:162 raises TypeError
    else status = RF_RANSAC_OK;
    if (status != RF_RANSAC_OK) {
        if (tid == 0) { *status_out = status; *nbInlier_out = 0; }
        for (int k = tid; k < 9; k += blockDim.x) H_out[k] = 0.f;
        for (int m = tid; m < M_host; m += blockDim.x) mask_out[m] = 0;
        return;
    }
    const unsigned best_i = 0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull);
    float H[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) H[k] = __ldcg(Hall + (long long)best_i * 9 + k);
    if (tid == 0) {
        *status_out = RF_RANSAC_OK;
        *nbInlier_out = (long long)(key >> 32);
    }
    if (tid < 9) H_out[tid] = H[tid];
    // utils/outil.py:162-163: recompute the inlier mask with the best H
    for (int m = tid; m < M_host; m += blockDim.x) {
        unsigned char v = 0;
        if (m < M) {
            float err = reproj_error(H, match1[m * 3], match1[m * 3 + 1], match2[m * 3], match2[m * 3 + 1], match2[m * 3 + 2]);
            v = (err < tol) ? 1 : 0;
        }
        mask_out[m] = v;
    }
}

__global__ void dlt_kernel(const float* __restrict__ X, const float* __restrict__ Y, int N, float* __restrict__ H_out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float xu[4], xv[4], yu[4], yv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        xu[k] = X[(i * 4 + k) * 3]; xv[k] = X[(i * 4 + k) * 3 + 1];
        yu[k] = Y[(i * 4 + k) * 3]; yv[k] = Y[(i * 4 + k) * 3 + 1];
    }
    float h[9];
    dlt_null_vector(xu, xv, yu, yv, h);
#pragma unroll
    for (int k = 0; k < 9; ++k) H_out[i * 9 + k] = h[k];
}

__global__ void prediction_kernel(const float* __restrict__ m1, const float* __restrict__ m2, int M,
                                  const float* __restrict__ Hs, int N, float* __restrict__ err) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)N * M) return;
    int n = (int)(t / M), m = (int)(t % M);
    float H[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) H[k] = Hs[n * 9 + k];
    err[t] = reproj_error(H, m1[m * 3], m1[m * 3 + 1], m2[m * 3], m2[m * 3 + 1], m2[m * 3 + 2]);
}

// gather matched coordinates (coarseAlignFeatMatch.py variant A :158-168 / variant C :146-155)
__global__ void build_matches_kernel(const long long* __restrict__ idx1, const long long* __restrict__ idx2,
                                     const int* __restrict__ count_in, const float* __restrict__ W1,
                                     const float* __restrict__ H1, const float* __restrict__ W2,
                                     const float* __restrict__ H2, const unsigned char* __restrict__ valid16,
                                     float* __restrict__ match1, float* __restrict__ match2,
                                     long long* __restrict__ idx2_kept, int* __restrict__ count_out, int capacity) {
    __shared__ int s_scan[32];
    __shared__ int s_off;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    const int n = min(*count_in, capacity);
    if (tid == 0) s_off = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
        int i = base + tid;
        long long a = 0, b = 0;
        int keep = 0;
        if (i < n) {
            a = idx1[i]; b = idx2[i];
            keep = (valid16 == nullptr) ? 1 : (valid16[b] != 0);
        }
        int incl = keep;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        int wofs = 0, total = 0;
        for (int w = 0; w < nw; ++w) { int v = s_scan[w]; if (w < warp) wofs += v; total += v; }
        int off = s_off;
        if (keep) {
            int o = off + wofs + incl - 1;
            match1[o * 3] = H1[a]; match1[o * 3 + 1] = W1[a]; match1[o * 3 + 2] = 1.0f;
            match2[o * 3] = H2[b]; match2[o * 3 + 1] = W2[b]; match2[o * 3 + 2] = 1.0f;
            if (idx2_kept) idx2_kept[o] = b;
        }
        __syncthreads();
        if (tid == 0) s_off = off + total;
        __syncthreads();
    }
    if (tid == 0) *count_out = s_off;
}

// evaluation/evalYFCC/evaluation.py:195-212 after the four RANSAC calls, as one CTA: per rotation k, drew = M_k >= nbPoint
// (the reference's getCoarse returns None before RANSAC otherwise), score = popcount(mask_k[:M_k]) when it drew and RANSAC
// returned a model (np.sum(InlierMask)), else 0; RF_RANSAC_NO_MODEL on a rotation that drew is utils/outil.py:162's TypeError;
// the winner is the first maximum (np.argmax).  Integer sums in a fixed order: deterministic, no atomics.
struct YfccSelectArgs {
    const int* status[4];
    const int* count[4];
    const unsigned char* mask[4];
    int cap[4];
};

constexpr int SELECT_THREADS = 256;

__global__ void __launch_bounds__(SELECT_THREADS)
yfcc_rotation_select_kernel(YfccSelectArgs a, int nbPoint, int* __restrict__ rec) {
    __shared__ int s_part[SELECT_THREADS / 32];
    __shared__ int s_score[4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int M = min(*a.count[k], a.cap[k]);
        const bool drew = M >= nbPoint;
        const bool ok = drew && *a.status[k] == RF_RANSAC_OK;
        int c = 0;
        if (ok)
            for (int m = tid; m < M; m += SELECT_THREADS) c += a.mask[k][m] != 0;
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) s_part[warp] = c;
        __syncthreads();
        if (tid == 0) {
            int t = 0;
#pragma unroll
            for (int w = 0; w < SELECT_THREADS / 32; ++w) t += s_part[w];
            s_score[k] = t;
        }
        __syncthreads();
    }
    if (tid == 0) {
        int best = 0, drawn = 0, err = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int M = min(*a.count[k], a.cap[k]);
            const bool drew = M >= nbPoint;
            drawn += drew ? 1 : 0;
            err |= (drew && *a.status[k] == RF_RANSAC_NO_MODEL) ? 1 : 0;
            if (s_score[k] > s_score[best]) best = k;
        }
        rec[RF_YFCC_REC_WINNER] = best;
#pragma unroll
        for (int k = 0; k < 4; ++k) rec[RF_YFCC_REC_SCORES + k] = s_score[k];
        rec[RF_YFCC_REC_DRAWN] = drawn;
        rec[RF_YFCC_REC_ERROR] = err;
        rec[RF_YFCC_REC_CLASS] = best & 1;
    }
}

// dst <- src[*sel] (nothing when that source is null): the winning rotation's buffers into the static ones a loop graph reads
struct SelectCopyArgs {
    const void* src[4];
};

__global__ void select_copy_kernel(SelectCopyArgs a, int nsrc, const int* __restrict__ sel, void* __restrict__ dst, size_t bytes,
                                   int vec16) {
    const int k = *sel;
    if (k < 0 || k >= nsrc) return;
    const void* src = k == 0 ? a.src[0] : k == 1 ? a.src[1] : k == 2 ? a.src[2] : a.src[3];     // constant indices: no local copy
    if (src == nullptr) return;
    const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
    if (vec16) {
        const uint4* s = static_cast<const uint4*>(src);
        uint4* d = static_cast<uint4*>(dst);
        for (size_t i = t0; i < bytes / 16; i += step) d[i] = s[i];
    } else {
        const unsigned char* s = static_cast<const unsigned char*>(src);
        unsigned char* d = static_cast<unsigned char*>(dst);
        for (size_t i = t0; i < bytes; i += step) d[i] = s[i];
    }
}

}  // namespace rf

using namespace rf;

extern "C" size_t rf_ransac_workspace(int nbIter) {
    size_t n = (size_t)(nbIter > 0 ? nbIter : 1);
    size_t b = 256;                       // header
    b += ((n * sizeof(int) + 255) / 256) * 256;          // counts
    b += ((n * 9 * sizeof(float) + 255) / 256) * 256;    // Hall
    b += ((n + 2) * sizeof(int) + 255) / 256 * 256;      // chunk_nz (chunk >= 1)
    return b;
}

static int launch_ransac(const float* match1, const float* match2, int M, const int* M_dev,
                         const int64_t* samples, int n_tables, int sample_mode, int nbIter, float tolerance, int chunk,
                         const int* slot_in, int* slot_out, float* H_out, int64_t* nbInlier_out, uint8_t* mask_out,
                         int* status_out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(M >= 0 && nbIter >= 0 && chunk >= 1 && n_tables >= 1, "rf_ransac_homography: bad sizes");
    RF_REQUIRE(sample_mode >= RF_SAMPLES_INDEX && sample_mode <= RF_SAMPLES_PHILOX64, "rf_ransac_homography: unknown sample_mode");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_ransac_workspace(nbIter), "rf_ransac_homography: workspace too small");
    RF_REQUIRE(slot_in != slot_out || slot_in == nullptr, "rf_ransac_homography_drawn: slot_in and slot_out must be two buffers");
    cudaStream_t st = as_stream(stream);
    size_t n = (size_t)(nbIter > 0 ? nbIter : 1);
    unsigned char* p = static_cast<unsigned char*>(ws);
    RansacHeader* hdr = reinterpret_cast<RansacHeader*>(p);
    p += 256;
    int* counts = reinterpret_cast<int*>(p);
    p += ((n * sizeof(int) + 255) / 256) * 256;
    float* Hall = reinterpret_cast<float*>(p);
    p += ((n * 9 * sizeof(float) + 255) / 256) * 256;
    int* chunk_nz = reinterpret_cast<int*>(p);
    RF_CUDA(cudaMemsetAsync(hdr, 0, sizeof(RansacHeader), st));
    const int sms = num_sms();
    int G = (nbIter >= 128 * 2 * sms) ? 128 : 32;
    int nGroups = (nbIter + G - 1) / G;
    int grid = nGroups < 1 ? 1 : (nGroups < 4 * sms ? nGroups : 4 * sms);
    size_t smem = (size_t)G * (9 * sizeof(float) + sizeof(int));
    ransac_kernel<<<grid, RANSAC_THREADS, smem, st>>>(match1, match2, M, M_dev, (const long long*)samples, sample_mode, nbIter, tolerance,
                                                      chunk, G, hdr, counts, Hall, chunk_nz, H_out,
                                                      (long long*)nbInlier_out, mask_out, status_out, slot_in, slot_out, n_tables);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_ransac_homography(const float* match1, const float* match2, int M, const int* M_dev,
                                    const int64_t* samples, int sample_mode, int nbIter, float tolerance, int chunk,
                                    float* H_out, int64_t* nbInlier_out, uint8_t* mask_out, int* status_out,
                                    void* ws, size_t ws_bytes, void* stream) {
    return launch_ransac(match1, match2, M, M_dev, samples, 1, sample_mode, nbIter, tolerance,
                         chunk, nullptr, nullptr, H_out, nbInlier_out, mask_out, status_out, ws, ws_bytes, stream);
}

extern "C" int rf_ransac_homography_drawn(const float* match1, const float* match2, int M, const int* M_dev,
                                          const int64_t* tables, int n_tables, int sample_mode, int nbIter, float tolerance,
                                          int chunk, const int* slot_in, int* slot_out, float* H_out, int64_t* nbInlier_out,
                                          uint8_t* mask_out, int* status_out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(slot_in != nullptr && slot_out != nullptr, "rf_ransac_homography_drawn: slot_in and slot_out are required");
    return launch_ransac(match1, match2, M, M_dev, tables, n_tables, sample_mode, nbIter,
                         tolerance, chunk, slot_in, slot_out, H_out, nbInlier_out, mask_out, status_out, ws, ws_bytes, stream);
}

extern "C" int rf_homography_dlt(const float* X, const float* Y, int N, float* H_out, void* stream) {
    if (N <= 0) return 0;
    const int threads = 64;
    dlt_kernel<<<(N + threads - 1) / threads, threads, 0, as_stream(stream)>>>(X, Y, N, H_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_prediction(const float* match1, const float* match2, int M, const float* H, int N, float* err_out, void* stream) {
    long long total = (long long)N * M;
    if (total <= 0) return 0;
    prediction_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(match1, match2, M, H, N, err_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_build_matches(const int64_t* idx1, const int64_t* idx2, const int* count_in,
                                const float* W1, const float* H1, const float* W2, const float* H2,
                                const uint8_t* valid16, float* match1_out, float* match2_out,
                                int64_t* idx2_kept_out, int* count_out, int capacity, void* stream) {
    build_matches_kernel<<<1, 256, 0, as_stream(stream)>>>((const long long*)idx1, (const long long*)idx2, count_in, W1, H1, W2, H2,
                                                            valid16, match1_out, match2_out, (long long*)idx2_kept_out,
                                                            count_out, capacity);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_yfcc_rotation_select(const int* const* status, const int* const* count, const uint8_t* const* mask, const int* cap,
                                       int nbPoint, int* rec_out, void* stream) {
    RF_REQUIRE(status != nullptr && count != nullptr && mask != nullptr && cap != nullptr && rec_out != nullptr,
               "rf_yfcc_rotation_select: null argument");
    RF_REQUIRE(nbPoint >= 1, "rf_yfcc_rotation_select: bad nbPoint");
    YfccSelectArgs a;
    for (int k = 0; k < 4; ++k) {
        RF_REQUIRE(status[k] != nullptr && count[k] != nullptr && cap[k] >= 0 && (mask[k] != nullptr || cap[k] == 0),
                   "rf_yfcc_rotation_select: bad rotation");
        a.status[k] = status[k];
        a.count[k] = count[k];
        a.mask[k] = mask[k];
        a.cap[k] = cap[k];
    }
    yfcc_rotation_select_kernel<<<1, SELECT_THREADS, 0, as_stream(stream)>>>(a, nbPoint, rec_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_select_copy(const void* const* src, int nsrc, const int* sel, void* dst, size_t bytes, void* stream) {
    RF_REQUIRE(src != nullptr && sel != nullptr && dst != nullptr && nsrc >= 1 && nsrc <= 4, "rf_select_copy: bad arguments");
    if (bytes == 0) return 0;
    SelectCopyArgs a;
    int vec16 = (bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) ? 1 : 0;
    for (int k = 0; k < 4; ++k) {
        a.src[k] = k < nsrc ? src[k] : nullptr;
        if (a.src[k] != nullptr && (reinterpret_cast<uintptr_t>(a.src[k]) & 15) != 0) vec16 = 0;
    }
    const size_t units = vec16 ? bytes / 16 : bytes;
    const size_t want = (units + 255) / 256;
    const int grid = (int)(want < (size_t)(4 * num_sms()) ? (want < 1 ? 1 : want) : (size_t)(4 * num_sms()));
    select_copy_kernel<<<grid, 256, 0, as_stream(stream)>>>(a, nsrc, sel, dst, bytes, vec16);
    RF_LAUNCHED();
    return 0;
}
