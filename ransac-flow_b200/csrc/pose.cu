// evalYFCC's relative-pose metric on the device (evaluation/evalYFCC/getResults.py:53-111):
//   rf_yfcc_matches      matches_from_flow + norm_kp (:29-71), order-preserving scan compaction;
//   rf_essential_ransac  cv2.findEssentialMat(RANSAC) (focal 1, pp (0, 0), prob 0.999, maxIters 1000): OpenCV's cv::RNG sample
//                        stream, a five-point solver per sample, the fp32-cast Sampson test and the sequential best-model replay;
//   rf_recover_pose      cv2.recoverPose over the stacked candidates, with the driver's strictly-greater loop.
// All fp64; the Sampson error and the match coordinates use explicit _rn intrinsics so that no FMA contraction changes them.
#include "common.cuh"

namespace rf {

constexpr int ESS_ITERS = 1000;          // maxIters of findEssentialMat
constexpr int ESS_BLOCK = 64;            // RANSAC iterations scored per launch
constexpr int ESS_NBLOCKS = (ESS_ITERS + ESS_BLOCK - 1) / ESS_BLOCK;
constexpr int ESS_MAXSOL = 10;
constexpr int SCORE_THREADS = 256;
constexpr int SCORE_PPT = 2;             // points per thread held in registers while looping over the block's models
constexpr int MATCH_TILE = 1024;         // mask elements per compaction tile

static inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// ------------------------------------------------------------------------------------------------------------ matches
__device__ __forceinline__ void rot_grid(int k, int i, int j, int wB, int hB, int& gx, int& gy) {
    // np.rot90(stack(meshgrid(arange(wB), arange(hB))), k)[i][j]; the unrotated grid holds (x = column, y = row)
    switch (k) {
    case 0: gx = j; gy = i; break;
    case 1: gx = wB - 1 - i; gy = j; break;
    case 2: gx = wB - 1 - j; gy = hB - 1 - i; break;
    default: gx = i; gy = hB - 1 - j; break;
    }
}

__global__ void match_count_kernel(const uint8_t* __restrict__ mask, long long P, int* __restrict__ tile_counts) {
    __shared__ int s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    const long long base = (long long)blockIdx.x * MATCH_TILE;
    int c = 0;
    for (int e = threadIdx.x; e < MATCH_TILE; e += blockDim.x) {
        const long long p = base + e;
        c += (p < P && mask[p] != 0) ? 1 : 0;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s, c);
    __syncthreads();
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = s;
}

// exclusive scan of the tile counts in one block (tiles <= a few thousand) + the total
__global__ void match_scan_kernel(int* __restrict__ tile_counts, int ntiles, int* __restrict__ N_out) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < ntiles; base += blockDim.x) {
        const int i = base + tid;
        const int v = i < ntiles ? tile_counts[i] : 0;
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        int wofs = 0, total = 0;
        for (int w = 0; w < nw; ++w) { const int x = s_warp[w]; if (w < warp) wofs += x; total += x; }
        const int carry = s_carry;
        if (i < ntiles) tile_counts[i] = carry + wofs + incl - v;
        __syncthreads();
        if (tid == 0) s_carry = carry + total;
        __syncthreads();
    }
    if (tid == 0) *N_out = s_carry;
}

__global__ void match_write_kernel(const float* __restrict__ flow, const uint8_t* __restrict__ mask, int H, int W, int k, int wB,
                                   int hB, float sxA, float syA, double4 n1, double4 n2, const int* __restrict__ tile_offsets,
                                   double* __restrict__ pts1, double* __restrict__ pts2) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const long long P = (long long)H * W;
    const long long base = (long long)blockIdx.x * MATCH_TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) s_carry = tile_offsets[blockIdx.x];
    __syncthreads();
    for (int e0 = 0; e0 < MATCH_TILE; e0 += blockDim.x) {
        const long long p = base + e0 + tid;
        const int keep = (p < P && mask[p] != 0) ? 1 : 0;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int wofs = 0, total = 0;
        for (int w = 0; w < nw; ++w) { const int x = s_warp[w]; if (w < warp) wofs += x; total += x; }
        const int carry = s_carry;
        if (keep) {
            const long long o = carry + wofs + __popc(bal & ((1u << lane) - 1u));
            const int i = (int)(p / W), j = (int)(p - (long long)i * W);
            // pts1 = flowFine[matchBinary]; pts1[:, 0] = (pts1[:, 0] + 1) * (wA - 1) / 2 in fp32 (no contraction), then norm_kp in fp64
            const float fx = __fdiv_rn(__fmul_rn(__fadd_rn(flow[2 * p], 1.0f), sxA), 2.0f);
            const float fy = __fdiv_rn(__fmul_rn(__fadd_rn(flow[2 * p + 1], 1.0f), syA), 2.0f);
            pts1[2 * o] = __ddiv_rn(__dsub_rn((double)fx, n1.x), n1.z);
            pts1[2 * o + 1] = __ddiv_rn(__dsub_rn((double)fy, n1.y), n1.w);
            int gx, gy;
            rot_grid(k, i, j, wB, hB, gx, gy);
            pts2[2 * o] = __ddiv_rn(__dsub_rn((double)gx, n2.x), n2.z);
            pts2[2 * o + 1] = __ddiv_rn(__dsub_rn((double)gy, n2.y), n2.w);
        }
        __syncthreads();
        if (tid == 0) s_carry = carry + total;
        __syncthreads();
    }
}

// ----------------------------------------------------------------------------------------------------- sample stream
__device__ void ess_reset(rf_pose_record_t* rec, int N) {
    rec->status = N < 5 ? RF_POSE_TOO_FEW : RF_POSE_OK;
    rec->n_points = N;
    rec->niters = ESS_ITERS;
    rec->best_iter = -1;
    rec->best_cand = -1;
    rec->ransac_count = 0;
    rec->n_E = 0;
    rec->pose_count = 0;
    rec->pose_cand = -1;
    rec->pose_index = -1;
    for (int c = 0; c < 4 * ESS_MAXSOL; ++c) rec->pose_counts[c] = 0;
}

// cv::RNG((uint64)-1): state = (uint32)state * 4164903690 + (state >> 32); uniform(0, N) = (uint32)state % N.
// RANSACPointSetRegistrator::getSubset redraws an index equal to one already in the subset; the essential-matrix callback
// accepts every subset, so one subset per iteration and the stream depends on N alone.
__global__ void ess_init_kernel(const int* __restrict__ N_dev, int* __restrict__ idx, rf_pose_record_t* __restrict__ rec) {
    const int N = *N_dev;
    if (rec) ess_reset(rec, N);
    if (N == 5) {
        for (int s = 0; s < 5; ++s) idx[s] = s;
        return;
    }
    if (N < 5) return;
    uint64_t state = ~0ull;
    for (int it = 0; it < ESS_ITERS; ++it) {
        int* d = idx + it * 5;
        for (int i = 0; i < 5; ++i) {
            for (;;) {
                state = (uint64_t)(uint32_t)state * 4164903690ull + (state >> 32);
                const int v = (int)((uint32_t)state % (uint32_t)N);
                int j = 0;
                while (j < i && d[j] != v) ++j;
                d[i] = v;
                if (j == i) break;
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------------- five-point
// Monomials of degree <= 3 in (x, y, z), code = 16 i + 4 j + k for x^i y^j z^k, mapped to the column order of the 10 x 20
// elimination: x3 y3 x2y xy2 x2z x2 y2z y2 xyz xy | xz2 xz x yz2 yz y z3 z2 z 1.  -1 = unused code.
__constant__ signed char c_col[64] = {
    // i = 0: j = 0..3, k = 0..3
    19, 18, 17, 16,   15, 14, 13, -1,   7, 6, -1, -1,   1, -1, -1, -1,
    // i = 1
    12, 11, 10, -1,   9, 8, -1, -1,   3, -1, -1, -1,   -1, -1, -1, -1,
    // i = 2
    5, 4, -1, -1,   2, -1, -1, -1,   -1, -1, -1, -1,   -1, -1, -1, -1,
    // i = 3
    0, -1, -1, -1,   -1, -1, -1, -1,   -1, -1, -1, -1,   -1, -1, -1, -1};
__constant__ unsigned char c_lin[4] = {16, 4, 1, 0};                               // x, y, z, 1
__constant__ unsigned char c_quad[10] = {32, 20, 17, 16, 8, 5, 4, 2, 1, 0};         // xx xy xz x yy yz y zz z 1

struct Quad { double c[10]; };   // coefficients over c_quad
struct Lin { double c[4]; };     // coefficients over c_lin

__device__ __forceinline__ int quad_slot(int code) {
    // position of a degree <= 2 code in c_quad
#pragma unroll
    for (int q = 0; q < 10; ++q)
        if (c_quad[q] == code) return q;
    return -1;
}

__device__ void lin_mul(const Lin& a, const Lin& b, Quad& out, double sgn) {
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) out.c[quad_slot(c_lin[u] + c_lin[v])] += sgn * a.c[u] * b.c[v];
}
__device__ void quad_lin_mul(const Quad& a, const Lin& b, double* row20, double sgn) {
#pragma unroll
    for (int u = 0; u < 10; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) row20[c_col[c_quad[u] + c_lin[v]]] += sgn * a.c[u] * b.c[v];
}

__device__ __forceinline__ double horner(const double* p, int d, double x) {
    double r = p[d];
    for (int i = d - 1; i >= 0; --i) r = r * x + p[i];
    return r;
}

// real roots of p (degree d <= 10, p[d] != 0) in ascending order: the roots of each derivative bracket the monotone pieces
// of the one above it (Gauss-Lucas keeps them inside the Cauchy bound of p); a piece whose ends differ in sign holds one
// root, found by bisection to the last bit.  Roots of even multiplicity (no sign change) are not reported.
__device__ int real_roots(const double* p, int d, double* roots) {
    double bound = 0.0;
    for (int i = 0; i < d; ++i) bound = fmax(bound, fabs(p[i] / p[d]));
    bound = 1.0 + bound;
    double crit[10];
    int ncrit = 0;
    double q[11];
    for (int level = d - 1; level >= 0; --level) {
        // q = p^(level), degree d - level
        const int dq = d - level;
        for (int i = 0; i <= dq; ++i) {
            double f = 1.0;
            for (int m = 1; m <= level; ++m) f *= (double)(i + m);
            q[i] = p[i + level] * f;
        }
        double found[10];
        int nf = 0;
        double a = -bound;
        double fa = horner(q, dq, a);
        for (int s = 0; s <= ncrit; ++s) {
            const double b = s < ncrit ? crit[s] : bound;
            const double fb = horner(q, dq, b);
            if (fa == 0.0) {
                if (nf == 0 || found[nf - 1] != a) found[nf++] = a;
            } else if ((fa < 0.0) != (fb < 0.0) && fb != 0.0) {
                double lo = a, hi = b, flo = fa;
                for (int it = 0; it < 2100; ++it) {
                    const double mid = 0.5 * (lo + hi);
                    if (mid <= lo || mid >= hi) break;
                    const double fm = horner(q, dq, mid);
                    if (fm == 0.0) { lo = hi = mid; break; }
                    if ((fm < 0.0) == (flo < 0.0)) { lo = mid; flo = fm; } else { hi = mid; }
                }
                found[nf++] = (fabs(horner(q, dq, lo)) <= fabs(horner(q, dq, hi))) ? lo : hi;
            }
            a = b;
            fa = fb;
        }
        if (fa == 0.0 && (nf == 0 || found[nf - 1] != a)) found[nf++] = a;
        ncrit = nf;
        for (int i = 0; i < nf; ++i) crit[i] = found[i];
    }
    for (int i = 0; i < ncrit; ++i) roots[i] = crit[i];
    return ncrit;
}

// polynomial products in z (coefficients by ascending power)
__device__ __forceinline__ void pmul(const double* a, int da, const double* b, int db, double* out) {
    for (int i = 0; i <= da + db; ++i) out[i] = 0.0;
    for (int i = 0; i <= da; ++i)
        for (int j = 0; j <= db; ++j) out[i + j] += a[i] * b[j];
}

// Solutions of x2^T E x1 = 0 at five correspondences with E essential: unit Frobenius norm, sign fixed so that the entry of
// largest magnitude is positive, in ascending order of the root z of the degree-10 polynomial.  Returns the count.
__device__ int five_point(const double (&x1)[5][2], const double (&x2)[5][2], double* Eout) {
    // null space of the 5 x 9 epipolar system: Householder QR of its transpose, basis = the last four columns of Q
    double A[9][5];
    for (int r = 0; r < 5; ++r) {
        const double u = x1[r][0], v = x1[r][1], s = x2[r][0], t = x2[r][1];
        A[0][r] = s * u; A[1][r] = s * v; A[2][r] = s;
        A[3][r] = t * u; A[4][r] = t * v; A[5][r] = t;
        A[6][r] = u; A[7][r] = v; A[8][r] = 1.0;
    }
    double V[5][9];   // Householder vectors
    double beta[5];
    for (int c = 0; c < 5; ++c) {
        double nrm = 0.0;
        for (int r = c; r < 9; ++r) nrm += A[r][c] * A[r][c];
        nrm = sqrt(nrm);
        const double alpha = A[c][c] >= 0.0 ? -nrm : nrm;
        for (int r = 0; r < 9; ++r) V[c][r] = r < c ? 0.0 : A[r][c];
        V[c][c] -= alpha;
        double vv = 0.0;
        for (int r = c; r < 9; ++r) vv += V[c][r] * V[c][r];
        beta[c] = vv > 0.0 ? 2.0 / vv : 0.0;
        for (int cc = c; cc < 5; ++cc) {
            double d = 0.0;
            for (int r = c; r < 9; ++r) d += V[c][r] * A[r][cc];
            d *= beta[c];
            for (int r = c; r < 9; ++r) A[r][cc] -= d * V[c][r];
        }
    }
    double basis[4][9];   // Q e_{5 + b} = H_0 H_1 ... H_4 e_{5 + b}
    for (int b = 0; b < 4; ++b) {
        double e[9];
        for (int r = 0; r < 9; ++r) e[r] = r == 5 + b ? 1.0 : 0.0;
        for (int c = 4; c >= 0; --c) {
            double d = 0.0;
            for (int r = c; r < 9; ++r) d += V[c][r] * e[r];
            d *= beta[c];
            for (int r = c; r < 9; ++r) e[r] -= d * V[c][r];
        }
        for (int r = 0; r < 9; ++r) basis[b][r] = e[r];
    }
    // E = x X + y Y + z Z + W: each entry a linear polynomial over (x, y, z, 1)
    Lin E[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            for (int b = 0; b < 4; ++b) E[i][j].c[b] = basis[b][3 * i + j];
    double M[10][20];
    for (int r = 0; r < 10; ++r)
        for (int c = 0; c < 20; ++c) M[r][c] = 0.0;
    // det E = 0
    {
        Quad cof;
        for (int u = 0; u < 10; ++u) cof.c[u] = 0.0;
        lin_mul(E[1][1], E[2][2], cof, 1.0); lin_mul(E[1][2], E[2][1], cof, -1.0);
        quad_lin_mul(cof, E[0][0], M[0], 1.0);
        for (int u = 0; u < 10; ++u) cof.c[u] = 0.0;
        lin_mul(E[1][0], E[2][2], cof, 1.0); lin_mul(E[1][2], E[2][0], cof, -1.0);
        quad_lin_mul(cof, E[0][1], M[0], -1.0);
        for (int u = 0; u < 10; ++u) cof.c[u] = 0.0;
        lin_mul(E[1][0], E[2][1], cof, 1.0); lin_mul(E[1][1], E[2][0], cof, -1.0);
        quad_lin_mul(cof, E[0][2], M[0], 1.0);
    }
    // (E E^T - tr(E E^T) / 2 I) E = 0
    {
        Quad EEt[3][3];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                for (int u = 0; u < 10; ++u) EEt[i][j].c[u] = 0.0;
                if (j < i) continue;
                for (int k = 0; k < 3; ++k) lin_mul(E[i][k], E[j][k], EEt[i][j], 1.0);
            }
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < i; ++j) EEt[i][j] = EEt[j][i];
        Quad half;
        for (int u = 0; u < 10; ++u) half.c[u] = 0.5 * (EEt[0][0].c[u] + EEt[1][1].c[u] + EEt[2][2].c[u]);
        for (int i = 0; i < 3; ++i)
            for (int u = 0; u < 10; ++u) EEt[i][i].c[u] -= half.c[u];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                for (int k = 0; k < 3; ++k) quad_lin_mul(EEt[i][k], E[k][j], M[1 + 3 * i + j], 1.0);
    }
    // Gauss-Jordan on the first ten columns (partial pivoting)
    for (int c = 0; c < 10; ++c) {
        int piv = c;
        for (int r = c + 1; r < 10; ++r)
            if (fabs(M[r][c]) > fabs(M[piv][c])) piv = r;
        if (M[piv][c] == 0.0) return 0;
        if (piv != c)
            for (int k = 0; k < 20; ++k) { const double t = M[c][k]; M[c][k] = M[piv][k]; M[piv][k] = t; }
        const double inv = 1.0 / M[c][c];
        for (int k = c; k < 20; ++k) M[c][k] *= inv;
        for (int r = 0; r < 10; ++r) {
            if (r == c) continue;
            const double f = M[r][c];
            if (f == 0.0) continue;
            for (int k = c; k < 20; ++k) M[r][k] -= f * M[c][k];
        }
    }
    // rows (x2z, x2), (y2z, y2), (xyz, xy): row_a - z row_b = 0 is linear in x, y with coefficients polynomial in z.
    // rest columns: 10 xz2, 11 xz, 12 x, 13 yz2, 14 yz, 15 y, 16 z3, 17 z2, 18 z, 19 1
    double B[3][3][5];
    for (int p = 0; p < 3; ++p) {
        const double* ra = M[4 + 2 * p];
        const double* rb = M[5 + 2 * p];
        B[p][0][0] = ra[12]; B[p][0][1] = ra[11] - rb[12]; B[p][0][2] = ra[10] - rb[11]; B[p][0][3] = -rb[10]; B[p][0][4] = 0.0;
        B[p][1][0] = ra[15]; B[p][1][1] = ra[14] - rb[15]; B[p][1][2] = ra[13] - rb[14]; B[p][1][3] = -rb[13]; B[p][1][4] = 0.0;
        B[p][2][0] = ra[19]; B[p][2][1] = ra[18] - rb[19]; B[p][2][2] = ra[17] - rb[18]; B[p][2][3] = ra[16] - rb[17];
        B[p][2][4] = -rb[16];
    }
    double poly[11];
    {
        double t1[8], t2[8], m1[7], m2[7], acc[11];
        for (int i = 0; i < 11; ++i) poly[i] = 0.0;
        // B00 (B11 B22 - B12 B21)
        pmul(B[1][1], 3, B[2][2], 4, t1); pmul(B[1][2], 4, B[2][1], 3, t2);
        for (int i = 0; i < 8; ++i) t1[i] -= t2[i];
        pmul(B[0][0], 3, t1, 7, acc);
        for (int i = 0; i < 11; ++i) poly[i] += acc[i];
        // - B01 (B10 B22 - B12 B20)
        pmul(B[1][0], 3, B[2][2], 4, t1); pmul(B[1][2], 4, B[2][0], 3, t2);
        for (int i = 0; i < 8; ++i) t1[i] -= t2[i];
        pmul(B[0][1], 3, t1, 7, acc);
        for (int i = 0; i < 11; ++i) poly[i] -= acc[i];
        // + B02 (B10 B21 - B11 B20)
        pmul(B[1][0], 3, B[2][1], 3, m1); pmul(B[1][1], 3, B[2][0], 3, m2);
        for (int i = 0; i < 7; ++i) m1[i] -= m2[i];
        pmul(B[0][2], 4, m1, 6, acc);
        for (int i = 0; i < 11; ++i) poly[i] += acc[i];
    }
    int deg = 10;
    while (deg > 0 && poly[deg] == 0.0) --deg;
    if (deg == 0) return 0;
    double zs[10];
    const int nz = real_roots(poly, deg, zs);
    int nsol = 0;
    for (int s = 0; s < nz; ++s) {
        const double z = zs[s];
        double Bz[3][3];
        for (int p = 0; p < 3; ++p)
            for (int q = 0; q < 3; ++q) Bz[p][q] = horner(B[p][q], q == 2 ? 4 : 3, z);
        // [x, y, 1] spans the null space of Bz: the largest cross product of two rows
        double best[3] = {0.0, 0.0, 0.0}, bn = -1.0;
        for (int a = 0; a < 3; ++a) {
            const int b = (a + 1) % 3;
            const double* r = Bz[a < b ? a : b];
            const double* t = Bz[a < b ? b : a];
            const double v[3] = {r[1] * t[2] - r[2] * t[1], r[2] * t[0] - r[0] * t[2], r[0] * t[1] - r[1] * t[0]};
            const double n = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
            if (n > bn) { bn = n; best[0] = v[0]; best[1] = v[1]; best[2] = v[2]; }
        }
        if (!(bn > 0.0) || best[2] == 0.0) continue;
        const double x = best[0] / best[2], y = best[1] / best[2];
        double e[9], n2 = 0.0;
        for (int k = 0; k < 9; ++k) {
            e[k] = x * basis[0][k] + y * basis[1][k] + z * basis[2][k] + basis[3][k];
            n2 += e[k] * e[k];
        }
        if (!(n2 > 0.0) || !isfinite(n2)) continue;
        const double inv = 1.0 / sqrt(n2);
        int km = 0;
        for (int k = 1; k < 9; ++k)
            if (fabs(e[k]) > fabs(e[km])) km = k;
        const double sg = e[km] < 0.0 ? -inv : inv;
        for (int k = 0; k < 9; ++k) Eout[9 * nsol + k] = e[k] * sg;
        ++nsol;
    }
    return nsol;
}

__global__ void __launch_bounds__(64) ess_solve_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                       const int* __restrict__ N_dev, const int* __restrict__ idx,
                                                       double* __restrict__ candE, int* __restrict__ ncand, int nsamples) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nsamples) return;
    const int N = N_dev ? *N_dev : 6;
    if (N < 5 || (N == 5 && s > 0)) { ncand[s] = 0; return; }
    double x1[5][2], x2[5][2];
    for (int i = 0; i < 5; ++i) {
        const int p = idx[5 * s + i];
        x1[i][0] = pts1[2 * p]; x1[i][1] = pts1[2 * p + 1];
        x2[i][0] = pts2[2 * p]; x2[i][1] = pts2[2 * p + 1];
    }
    ncand[s] = five_point(x1, x2, candE + (size_t)s * ESS_MAXSOL * 9);
}

// --------------------------------------------------------------------------------------------------------- scoring
// EMEstimatorCallback::computeError in its operation order, no contraction: (float)(r^2 / (Ex1_0^2 + Ex1_1^2 + Etx2_0^2 + Etx2_1^2))
__device__ __forceinline__ float sampson(const double* E, double u1, double v1, double u2, double v2) {
    const double ex0 = __dadd_rn(__dadd_rn(__dmul_rn(E[0], u1), __dmul_rn(E[1], v1)), E[2]);
    const double ex1 = __dadd_rn(__dadd_rn(__dmul_rn(E[3], u1), __dmul_rn(E[4], v1)), E[5]);
    const double ex2 = __dadd_rn(__dadd_rn(__dmul_rn(E[6], u1), __dmul_rn(E[7], v1)), E[8]);
    const double et0 = __dadd_rn(__dadd_rn(__dmul_rn(E[0], u2), __dmul_rn(E[3], v2)), E[6]);
    const double et1 = __dadd_rn(__dadd_rn(__dmul_rn(E[1], u2), __dmul_rn(E[4], v2)), E[7]);
    const double r = __dadd_rn(__dadd_rn(__dmul_rn(u2, ex0), __dmul_rn(v2, ex1)), ex2);
    const double den = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex0, ex0), __dmul_rn(ex1, ex1)), __dmul_rn(et0, et0)), __dmul_rn(et1, et1));
    return __double2float_rn(__ddiv_rn(__dmul_rn(r, r), den));
}

// counts[m] += inliers of model m over the points; models = the candidates of iterations [it0, it0 + ESS_BLOCK) (or an
// explicit list when `it0 < 0`: nmodels models at E, used by rf_essential_score).  A block whose first iteration is at or
// beyond the replay's current iteration budget exits at once.
__global__ void __launch_bounds__(SCORE_THREADS) ess_score_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                                  const int* __restrict__ N_dev, int N_host, int it0,
                                                                  const double* __restrict__ E, const int* __restrict__ ncand,
                                                                  int nmodels, int* __restrict__ counts, float* __restrict__ err_out,
                                                                  const rf_pose_record_t* __restrict__ rec, float thr2) {
    extern __shared__ double s_E[];                         // [ESS_BLOCK * ESS_MAXSOL][9]
    __shared__ int s_slot[ESS_BLOCK * ESS_MAXSOL];          // counts index of each compacted model
    __shared__ int s_cnt[ESS_BLOCK * ESS_MAXSOL];
    __shared__ int s_m;
    const int N = N_dev ? *N_dev : N_host;
    if (it0 >= 0 && (N <= 5 || it0 >= rec->niters)) return;
    // the grid covers the buffer's capacity (H * W of the target on the metric's path); only the first N points are matches
    if ((long long)blockIdx.x * SCORE_PPT * blockDim.x >= N) return;
    const int tid = threadIdx.x;
    if (tid == 0) {
        int m = 0;
        if (it0 >= 0) {
            for (int it = it0; it < it0 + ESS_BLOCK && it < ESS_ITERS; ++it)
                for (int c = 0; c < ncand[it]; ++c) s_slot[m++] = it * ESS_MAXSOL + c;
        } else {
            for (; m < nmodels; ++m) s_slot[m] = m;
        }
        s_m = m;
    }
    __syncthreads();
    const int M = s_m;
    for (int e = tid; e < M * 9; e += blockDim.x) s_E[e] = E[(size_t)s_slot[e / 9] * 9 + e % 9];
    for (int e = tid; e < M; e += blockDim.x) s_cnt[e] = 0;
    __syncthreads();
    double u1[SCORE_PPT], v1[SCORE_PPT], u2[SCORE_PPT], v2[SCORE_PPT];
    bool ok[SCORE_PPT];
    long long pidx[SCORE_PPT];
#pragma unroll
    for (int q = 0; q < SCORE_PPT; ++q) {
        const long long p = ((long long)blockIdx.x * SCORE_PPT + q) * blockDim.x + tid;
        pidx[q] = p;
        ok[q] = p < N;
        u1[q] = ok[q] ? pts1[2 * p] : 0.0; v1[q] = ok[q] ? pts1[2 * p + 1] : 0.0;
        u2[q] = ok[q] ? pts2[2 * p] : 0.0; v2[q] = ok[q] ? pts2[2 * p + 1] : 0.0;
    }
    for (int m = 0; m < M; ++m) {
        int c = 0;
#pragma unroll
        for (int q = 0; q < SCORE_PPT; ++q) {
            const float err = sampson(s_E + 9 * m, u1[q], v1[q], u2[q], v2[q]);
            c += __popc(__ballot_sync(0xffffffffu, ok[q] && err <= thr2));
            if (err_out && ok[q]) err_out[(size_t)m * N + pidx[q]] = err;
        }
        if ((tid & 31) == 0 && c) atomicAdd(&s_cnt[m], c);
    }
    __syncthreads();
    for (int e = tid; e < M; e += blockDim.x)
        if (s_cnt[e]) atomicAdd(&counts[s_slot[e]], s_cnt[e]);
}

// RANSACUpdateNumIters(p, ep, modelPoints, maxIters).  CUDA's pow / log are within an ulp or two of glibc's, not always equal
// to them: the rounded budget can differ from OpenCV's only when num / denom lies within a few ulps of a .5 boundary.  The
// end-to-end tests compare the budget with the host oracle's (numpy, glibc) on every scene.
__device__ int update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = fmin(fmax(p, 0.0), 1.0);
    ep = fmin(fmax(ep, 0.0), 1.0);
    double num = fmax(1.0 - p, 2.2250738585072014e-308);
    double denom = 1.0 - pow(1.0 - ep, (double)model_points);
    if (denom < 2.2250738585072014e-308) return 0;
    num = log(num);
    denom = log(denom);
    return (denom >= 0.0 || -num >= max_iters * (-denom)) ? max_iters : __double2int_rn(num / denom);
}

// RANSACPointSetRegistrator::run's sequential part for iterations [it0, it0 + ESS_BLOCK): a candidate replaces the best when
// its count exceeds max(best, 4); each replacement shrinks the iteration budget.
__global__ void ess_replay_kernel(int it0, const int* __restrict__ ncand, const int* __restrict__ counts, rf_pose_record_t* __restrict__ rec) {
    const int N = rec->n_points;
    if (N <= 5) return;
    int niters = rec->niters, best = rec->ransac_count, bi = rec->best_iter, bc = rec->best_cand;
    for (int it = it0; it < it0 + ESS_BLOCK && it < niters; ++it) {
        for (int c = 0; c < ncand[it]; ++c) {
            const int cnt = counts[it * ESS_MAXSOL + c];
            if (cnt > max(best, 4)) {
                best = cnt; bi = it; bc = c;
                niters = update_num_iters(0.999, (double)(N - cnt) / N, 5, niters);
            }
        }
    }
    rec->niters = niters;
    rec->ransac_count = best;
    rec->best_iter = bi;
    rec->best_cand = bc;
}

// the best model's mask; block 0 fills the record (E, status)
__global__ void ess_final_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2, int capacity,
                                 const double* __restrict__ candE, const int* __restrict__ ncand, rf_pose_record_t* __restrict__ rec,
                                 float thr2, uint8_t* __restrict__ mask_out) {
    const int N = rec->n_points;
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int bi = rec->best_iter, bc = rec->best_cand;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (N < 5) {
            rec->status = RF_POSE_TOO_FEW;
        } else if (N == 5) {
            rec->n_E = ncand[0];
            for (int k = 0; k < ncand[0] * 9; ++k) rec->E[k] = candE[k];
            rec->status = ncand[0] > 0 ? RF_POSE_OK : RF_POSE_NO_MODEL;
            rec->ransac_count = ncand[0] > 0 ? 5 : 0;
        } else if (bi < 0) {
            rec->status = RF_POSE_NO_MODEL;
        } else {
            rec->n_E = 1;
            for (int k = 0; k < 9; ++k) rec->E[k] = candE[((size_t)bi * ESS_MAXSOL + bc) * 9 + k];
        }
    }
    if (p >= N || p >= capacity) return;
    uint8_t m = 0;
    if (N == 5) m = ncand[0] > 0 ? 1 : 0;
    else if (N > 5 && bi >= 0)
        m = sampson(candE + ((size_t)bi * ESS_MAXSOL + bc) * 9, pts1[2 * p], pts1[2 * p + 1], pts2[2 * p], pts2[2 * p + 1]) <= thr2;
    mask_out[p] = m;
}

// ------------------------------------------------------------------------------------------------------ recoverPose
// one-sided Jacobi SVD of an n x n matrix (n <= 4, columns of a): on return the columns of v are the right singular vectors
// and the columns of a are u_i * sigma_i
template <int n>
__device__ __forceinline__ void jacobi_svd(double (&a)[n][n], double (&v)[n][n]) {
#pragma unroll
    for (int i = 0; i < n; ++i)
#pragma unroll
        for (int j = 0; j < n; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; ++sweep) {
        bool rotated = false;
#pragma unroll
        for (int i = 0; i < n - 1; ++i)
#pragma unroll
            for (int j = i + 1; j < n; ++j) {
                double al = 0.0, be = 0.0, ga = 0.0;
#pragma unroll
                for (int r = 0; r < n; ++r) { al += a[r][i] * a[r][i]; be += a[r][j] * a[r][j]; ga += a[r][i] * a[r][j]; }
                if (ga == 0.0 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
                for (int r = 0; r < n; ++r) {
                    const double x = a[r][i], y = a[r][j];
                    a[r][i] = c * x - s * y; a[r][j] = s * x + c * y;
                    const double p = v[r][i], q = v[r][j];
                    v[r][i] = c * p - s * q; v[r][j] = s * p + c * q;
                }
            }
        if (!rotated) break;
    }
}

__device__ __forceinline__ double det3(const double (&m)[3][3]) {
    return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

// decomposeEssentialMat per candidate: E = U S V^T (det fixes: U *= -1, V *= -1), R1 = U W V^T, R2 = U W^T V^T, t = U_3;
// poses in OpenCV's order (R1, t), (R2, t), (R1, -t), (R2, -t), each [R row-major | t]
__global__ void pose_decompose_kernel(rf_pose_record_t* __restrict__ rec) {
    const int c = threadIdx.x;
    if (c == 0)
        for (int k = 0; k < 4 * ESS_MAXSOL; ++k) rec->pose_counts[k] = 0;
    if (c >= rec->n_E) return;
    double a[3][3], v[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) a[i][j] = rec->E[9 * c + 3 * i + j];
    jacobi_svd<3>(a, v);
    double sg[3];
    for (int j = 0; j < 3; ++j) sg[j] = sqrt(a[0][j] * a[0][j] + a[1][j] * a[1][j] + a[2][j] * a[2][j]);
    int o[3] = {0, 1, 2};   // descending singular values
    for (int i = 0; i < 3; ++i)
        for (int j = i + 1; j < 3; ++j)
            if (sg[o[j]] > sg[o[i]]) { const int t = o[i]; o[i] = o[j]; o[j] = t; }
    double U[3][3], Vm[3][3];
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) Vm[r][k] = v[r][o[k]];
    for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 3; ++r) U[r][k] = a[r][o[k]] / sg[o[k]];
    // U_3: the unit vector orthogonal to U_1, U_2 (E's left null vector)
    U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
    U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
    U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
    {
        const double n = sqrt(U[0][2] * U[0][2] + U[1][2] * U[1][2] + U[2][2] * U[2][2]);
        for (int r = 0; r < 3; ++r) U[r][2] /= n;
    }
    if (det3(U) < 0.0)
        for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) U[r][k] = -U[r][k];
    if (det3(Vm) < 0.0)
        for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) Vm[r][k] = -Vm[r][k];
    // R1 = U W V^T with W = [[0, 1, 0], [-1, 0, 0], [0, 0, 1]]: U W = [-U_2, U_1, U_3]; R2: U W^T = [U_2, -U_1, U_3]
    double R1[3][3], R2[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            R1[i][j] = -U[i][1] * Vm[j][0] + U[i][0] * Vm[j][1] + U[i][2] * Vm[j][2];
            R2[i][j] = U[i][1] * Vm[j][0] - U[i][0] * Vm[j][1] + U[i][2] * Vm[j][2];
        }
    for (int p = 0; p < 4; ++p) {
        double* P = rec->poses + (4 * c + p) * 12;
        const double (&R)[3][3] = (p & 1) ? R2 : R1;
        const double ts = p < 2 ? 1.0 : -1.0;
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) P[4 * i + j] = R[i][j];
            P[4 * i + 3] = ts * U[i][2];
        }
    }
}

// cv::triangulatePoints (null vector of the 4 x 4 DLT system) + recoverPose's cheirality test for every pose of every
// candidate: bit 4 c + p of bits[i] = point i in front of both cameras of pose p of candidate c, closer than 50.  The counts
// of candidate 0 (ANDed with mask_in) are block-reduced into pose_counts; no triangulated point leaves registers.
__device__ __forceinline__ bool cheiral(const double* P, double x1, double y1, double x2, double y2) {
    double A[4][4];
    A[0][0] = -1.0; A[0][1] = 0.0; A[0][2] = x1; A[0][3] = 0.0;
    A[1][0] = 0.0; A[1][1] = -1.0; A[1][2] = y1; A[1][3] = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        A[2][k] = x2 * P[8 + k] - P[k];
        A[3][k] = y2 * P[8 + k] - P[4 + k];
    }
    double V[4][4];
    jacobi_svd<4>(A, V);
    int jm = 0;
    double nm = 1e308;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const double n = A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j] + A[3][j] * A[3][j];
        if (n < nm) { nm = n; jm = j; }
    }
    double Q[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) Q[r] = V[r][jm];
    bool ok = Q[2] * Q[3] > 0.0;
    const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3], Wn = Q[3] / Q[3];
    ok = ok && Z < 50.0;
    const double z2 = P[8] * X + P[9] * Y + P[10] * Z + P[11] * Wn;
    return ok && z2 > 0.0 && z2 < 50.0;
}

__global__ void __launch_bounds__(256) pose_cheirality_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                              int capacity, const uint8_t* __restrict__ mask_in,
                                                              rf_pose_record_t* __restrict__ rec, unsigned long long* __restrict__ bits) {
    __shared__ double s_P[4 * ESS_MAXSOL * 12];
    __shared__ int s_cnt[4];
    const int N = rec->n_points, nE = rec->n_E;
    if (rec->status != RF_POSE_OK || (long long)blockIdx.x * blockDim.x >= N) return;
    for (int e = threadIdx.x; e < 4 * nE * 12; e += blockDim.x) s_P[e] = rec->poses[e];
    if (threadIdx.x < 4) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < N && i < capacity;
    const double x1 = live ? pts1[2 * i] : 0.0, y1 = live ? pts1[2 * i + 1] : 0.0;
    const double x2 = live ? pts2[2 * i] : 0.0, y2 = live ? pts2[2 * i + 1] : 0.0;
    const bool m = live && mask_in[i] != 0;
    unsigned long long b = 0;
    for (int c = 0; c < nE; ++c)
        for (int p = 0; p < 4; ++p) {
            const bool g = live && cheiral(s_P + (4 * c + p) * 12, x1, y1, x2, y2);
            if (g) b |= 1ull << (4 * c + p);
            if (c == 0) {
                const int n = __popc(__ballot_sync(0xffffffffu, g && m));
                if ((threadIdx.x & 31) == 0 && n) atomicAdd(&s_cnt[p], n);
            }
        }
    if (live) bits[i] = b;
    __syncthreads();
    if (threadIdx.x < 4 && s_cnt[threadIdx.x]) atomicAdd(&rec->pose_counts[threadIdx.x], s_cnt[threadIdx.x]);
}

// recoverPose's choice (good1 >= ... in pose order) per candidate, then the driver's loop over the stacked candidates:
// cv2 writes each call's mask into the array passed as mask=, so candidate c + 1 sees candidate c's output mask, and the
// first candidate with the strictly largest count wins.  Candidates after the first (only the five-point case stacks
// them) are recounted here in one block.
__global__ void pose_select_kernel(const uint8_t* __restrict__ mask_in, int capacity, rf_pose_record_t* __restrict__ rec,
                                   const unsigned long long* __restrict__ bits, uint8_t* __restrict__ chain,
                                   uint8_t* __restrict__ mask_out) {
    __shared__ int s_cnt[4];
    __shared__ int s_pick;
    if (rec->status != RF_POSE_OK) return;
    const int N = min(rec->n_points, capacity), nE = rec->n_E;
    int best = 0, bc = -1, bp = -1;
    for (int c = 0; c < nE; ++c) {
        if (threadIdx.x < 4) s_cnt[threadIdx.x] = c == 0 ? rec->pose_counts[threadIdx.x] : 0;
        __syncthreads();
        if (c > 0) {
            for (int i = threadIdx.x; i < N; i += blockDim.x)
                if (chain[i])
                    for (int p = 0; p < 4; ++p)
                        if ((bits[i] >> (4 * c + p)) & 1ull) atomicAdd(&s_cnt[p], 1);
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            const int g1 = s_cnt[0], g2 = s_cnt[1], g3 = s_cnt[2], g4 = s_cnt[3];
            int p;
            if (g1 >= g2 && g1 >= g3 && g1 >= g4) p = 0;
            else if (g2 >= g1 && g2 >= g3 && g2 >= g4) p = 1;
            else if (g3 >= g1 && g3 >= g2 && g3 >= g4) p = 2;
            else p = 3;
            if (c > 0) for (int q = 0; q < 4; ++q) rec->pose_counts[4 * c + q] = s_cnt[q];
            s_pick = p;
        }
        __syncthreads();
        const int p = s_pick, g = s_cnt[p];
        // this candidate's output mask becomes the next candidate's input (and is the answer if it wins)
        if (nE > 1)
            for (int i = threadIdx.x; i < N; i += blockDim.x) {
                const uint8_t in = c == 0 ? (mask_in[i] != 0) : chain[i];
                const uint8_t out = in && ((bits[i] >> (4 * c + p)) & 1ull);
                chain[i] = out;
                if (g > best) mask_out[i] = out;
            }
        if (g > best) { best = g; bc = c; bp = p; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        rec->pose_count = best;
        rec->pose_cand = bc;
        rec->pose_index = bp;
        if (bc < 0) {
            rec->status = RF_POSE_NO_POSE;
        } else {
            const double* P = rec->poses + (4 * bc + bp) * 12;
            for (int r = 0; r < 3; ++r) {
                for (int k = 0; k < 3; ++k) rec->R[3 * r + k] = P[4 * r + k];
                rec->t[r] = P[4 * r + 3];
            }
        }
    }
}

// single-candidate mask: the chosen pose's bits ANDed with the input mask.  Every other outcome that pose_select_kernel
// left unwritten (no stacked candidate won, or no E to start from) gets zeros: what cv2's mask= array holds when every count is 0
__global__ void pose_mask_kernel(const uint8_t* __restrict__ mask_in, int capacity, const rf_pose_record_t* __restrict__ rec,
                                 const unsigned long long* __restrict__ bits, uint8_t* __restrict__ mask_out) {
    if (rec->n_E > 1 && rec->status == RF_POSE_OK) return;   // the winner's chained mask, written by pose_select_kernel
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rec->n_points || i >= capacity) return;
    const int p = rec->pose_index;
    mask_out[i] = (rec->status == RF_POSE_OK && p >= 0) ? (uint8_t)(mask_in[i] != 0 && ((bits[i] >> p) & 1ull)) : 0;
}

// ------------------------------------------------------------------------------------------------ findFundamentalMat
// cv2.findFundamentalMat(FM_8POINT): run8Point (N >= 8) / run7Point (N == 7) on the points cast to fp32.  Three passes over
// the points (centroids, mean distances, the 45 moments); each CTA writes its partial sums, and every consumer sums the
// partials of the CTAs that held points in the same fixed order, so the result does not depend on scheduling.
constexpr int FM_THREADS = 256;
constexpr int FM_MAXGRID = 512;
constexpr int FM_STATS = 51;             // m1c (2), m2c (2), scale1, scale2, A's upper triangle (45)

static inline int fm_grid(int capacity) {
    const int g = (capacity + FM_THREADS - 1) / FM_THREADS;
    return g < 1 ? 1 : (g > FM_MAXGRID ? FM_MAXGRID : g);
}

struct FmWs {
    double* p1;   // [grid][4]  sum of (x1, y1, x2, y2)
    double* p2;   // [grid][2]  sum of the distances to the centroids
    double* p3;   // [grid][45] sum of r r^T
};
static FmWs fm_carve(void* ws, int grid) {
    unsigned char* p = static_cast<unsigned char*>(ws);
    FmWs w;
    w.p1 = reinterpret_cast<double*>(p);
    p += align256((size_t)grid * 4 * sizeof(double));
    w.p2 = reinterpret_cast<double*>(p);
    p += align256((size_t)grid * 2 * sizeof(double));
    w.p3 = reinterpret_cast<double*>(p);
    return w;
}

// findFundamentalMat's convertTo(CV_32F), back in fp64 for run8Point's arithmetic
__device__ __forceinline__ void fm_load(const double* __restrict__ pts1, const double* __restrict__ pts2, long long i, double& x1,
                                        double& y1, double& x2, double& y2) {
    x1 = (double)__double2float_rn(pts1[2 * i]);
    y1 = (double)__double2float_rn(pts1[2 * i + 1]);
    x2 = (double)__double2float_rn(pts2[2 * i]);
    y2 = (double)__double2float_rn(pts2[2 * i + 1]);
}

// the CTA's sums of v[K] into out[K]: xor-butterfly within each warp, then the warps in order
template <int K>
__device__ __forceinline__ void fm_block_sum(double (&v)[K], double* __restrict__ out) {
    __shared__ double s[FM_THREADS / 32][K];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double x = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) s[warp][k] = x;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        double x = 0.0;
        for (int w = 0; w < FM_THREADS / 32; ++w) x += s[w][k];
        out[k] = x;
    }
}

// sum over the first `active` CTAs' partials part[g][K] (component k) in one warp: lanes stride over g, then an xor
// butterfly; every lane, and every CTA that calls it, gets the same bits
__device__ __forceinline__ double fm_warp_total(const double* __restrict__ part, int K, int k, int active) {
    double x = 0.0;
    for (int g = threadIdx.x & 31; g < active; g += 32) x += part[(size_t)g * K + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

__device__ __forceinline__ int fm_active(int N, int grid) {
    const int a = (N + FM_THREADS - 1) / FM_THREADS;
    return a < grid ? a : grid;
}

// centroids (cv: m1c += Point2d(m1[i]); m1c *= 1. / count) from the pass-1 partials, by warp 0 of the calling CTA
__device__ __forceinline__ void fm_centroids(const FmWs& w, int N, int grid, double* __restrict__ c) {
    const int active = fm_active(N, grid);
    const double t = 1.0 / N;
    for (int k = 0; k < 4; ++k) {
        const double s = fm_warp_total(w.p1, 4, k, active);
        if (threadIdx.x == 0) c[k] = s * t;
    }
}

// scale = sqrt(2) / mean distance; a mean below FLT_EPSILON marks a degenerate set (returned as scale 0)
__device__ __forceinline__ void fm_scales(const FmWs& w, int N, int grid, double* __restrict__ sc) {
    const int active = fm_active(N, grid);
    const double t = 1.0 / N;
    for (int k = 0; k < 2; ++k) {
        const double m = fm_warp_total(w.p2, 2, k, active) * t;
        if (threadIdx.x == 0) sc[k] = m < 1.1920928955078125e-07 ? 0.0 : 1.4142135623730951 / m;
    }
}

// pass 1: centroid sums; also writes the all-ones mask of findFundamentalMat when N >= 7
__global__ void __launch_bounds__(FM_THREADS) fm_centroid_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                                 const int* __restrict__ N_dev, FmWs w, uint8_t* __restrict__ mask_out) {
    const int N = *N_dev;
    if ((long long)blockIdx.x * FM_THREADS >= N) return;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long i = (long long)blockIdx.x * FM_THREADS + threadIdx.x; i < N; i += (long long)gridDim.x * FM_THREADS) {
        double x1, y1, x2, y2;
        fm_load(pts1, pts2, i, x1, y1, x2, y2);
        v[0] += x1; v[1] += y1; v[2] += x2; v[3] += y2;
        if (mask_out && N >= 7) mask_out[i] = 1;
    }
    fm_block_sum<4>(v, w.p1 + (size_t)blockIdx.x * 4);
}

// pass 2: sums of the distances to the centroids
__global__ void __launch_bounds__(FM_THREADS) fm_distance_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                                 const int* __restrict__ N_dev, FmWs w) {
    __shared__ double s_c[4];
    const int N = *N_dev;
    if ((long long)blockIdx.x * FM_THREADS >= N) return;
    if (threadIdx.x < 32) fm_centroids(w, N, gridDim.x, s_c);
    __syncthreads();
    const double c0 = s_c[0], c1 = s_c[1], c2 = s_c[2], c3 = s_c[3];
    double v[2] = {0.0, 0.0};
    for (long long i = (long long)blockIdx.x * FM_THREADS + threadIdx.x; i < N; i += (long long)gridDim.x * FM_THREADS) {
        double x1, y1, x2, y2;
        fm_load(pts1, pts2, i, x1, y1, x2, y2);
        const double a = x1 - c0, b = y1 - c1, d = x2 - c2, e = y2 - c3;
        v[0] += sqrt(a * a + b * b);
        v[1] += sqrt(d * d + e * e);
    }
    fm_block_sum<2>(v, w.p2 + (size_t)blockIdx.x * 2);
}

// r = (x2 x1, x2 y1, x2, y2 x1, y2 y1, y2, x1, y1, 1) of a normalised point pair
__device__ __forceinline__ void fm_row(double x1, double y1, double x2, double y2, const double* c, const double* sc, double (&r)[9]) {
    const double u1 = (x1 - c[0]) * sc[0], v1 = (y1 - c[1]) * sc[0];
    const double u2 = (x2 - c[2]) * sc[1], v2 = (y2 - c[3]) * sc[1];
    r[0] = u2 * u1; r[1] = u2 * v1; r[2] = u2;
    r[3] = v2 * u1; r[4] = v2 * v1; r[5] = v2;
    r[6] = u1; r[7] = v1; r[8] = 1.0;
}

// pass 3: the 45 distinct sums of r r^T
__global__ void __launch_bounds__(FM_THREADS, 1) fm_moment_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                               const int* __restrict__ N_dev, FmWs w) {
    __shared__ double s_c[4], s_sc[2];
    const int N = *N_dev;
    if ((long long)blockIdx.x * FM_THREADS >= N) return;
    if (threadIdx.x < 32) {
        fm_centroids(w, N, gridDim.x, s_c);
        fm_scales(w, N, gridDim.x, s_sc);
    }
    __syncthreads();
    const double c[4] = {s_c[0], s_c[1], s_c[2], s_c[3]}, sc[2] = {s_sc[0], s_sc[1]};
    double acc[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) acc[k] = 0.0;
    for (long long i = (long long)blockIdx.x * FM_THREADS + threadIdx.x; i < N; i += (long long)gridDim.x * FM_THREADS) {
        double x1, y1, x2, y2, r[9];
        fm_load(pts1, pts2, i, x1, y1, x2, y2);
        fm_row(x1, y1, x2, y2, c, sc, r);
        int k = 0;
#pragma unroll
        for (int a = 0; a < 9; ++a)
#pragma unroll
            for (int b = a; b < 9; ++b) acc[k++] += r[a] * r[b];
    }
    fm_block_sum<45>(acc, w.p3 + (size_t)blockIdx.x * 45);
}

// the statistics run8Point works from, by one warp: out[FM_STATS] as rf_fundamental_moments documents
__device__ void fm_stats(const FmWs& w, int N, int grid, double* __restrict__ out) {
    fm_centroids(w, N, grid, out);
    fm_scales(w, N, grid, out + 4);
    const int active = fm_active(N, grid);
    for (int k = 0; k < 45; ++k) {
        const double s = fm_warp_total(w.p3, 45, k, active);
        if (threadIdx.x == 0) out[6 + k] = s;
    }
}

__global__ void fm_stats_kernel(const int* __restrict__ N_dev, FmWs w, int grid, double* __restrict__ out) {
    const int N = *N_dev;
    if (N >= 1) fm_stats(w, N, grid, out);
}

// the eigen-decomposition of the symmetric 9 x 9 A by one warp: one-sided Jacobi (the SVD of A, whose right vectors are A's
// eigenvectors) with lane j < 9 holding column j of A and of V, the nine columns paired round-robin (9 rounds of four
// disjoint pairs per sweep).  On return lam = v_j . a_j, the signed eigenvalue of lane j, and v = its eigenvector.
__device__ void fm_eigen9(double (&a)[9], double (&v)[9], double& lam) {
    const int j = threadIdx.x & 31;
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int round = 0; round < 9; ++round) {
            const int p = j < 9 ? (2 * round - j + 18) % 9 : j;   // partner; p == j: idle this round
            double ap[9], vp[9];
#pragma unroll
            for (int r = 0; r < 9; ++r) {
                ap[r] = __shfl_sync(0xffffffffu, a[r], p);
                vp[r] = __shfl_sync(0xffffffffu, v[r], p);
            }
            if (p == j) continue;
            const bool lo = j < p;                                  // this lane holds column i of the pair (i < k)
            double ni = 0.0, nk = 0.0, g = 0.0;
#pragma unroll
            for (int r = 0; r < 9; ++r) {
                const double ai = lo ? a[r] : ap[r], ak = lo ? ap[r] : a[r];
                ni += ai * ai; nk += ak * ak; g += ai * ak;
            }
            if (g == 0.0 || fabs(g) <= 2.220446049250313e-16 * sqrt(ni * nk)) continue;
            rotated = true;
            const double zeta = (nk - ni) / (2.0 * g);
            const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
            for (int r = 0; r < 9; ++r) {
                // column i -> c a_i - s a_k, column k -> s a_i + c a_k
                a[r] = lo ? c * a[r] - s * ap[r] : s * ap[r] + c * a[r];
                v[r] = lo ? c * v[r] - s * vp[r] : s * vp[r] + c * v[r];
            }
        }
        if (!__any_sync(0xffffffffu, rotated)) break;
    }
    lam = 0.0;
#pragma unroll
    for (int r = 0; r < 9; ++r) lam += a[r] * v[r];
}

// F = T2^T F0 T1 with T = [[s, 0, -s cx], [0, s, -s cy], [0, 0, 1]], then F *= 1 / F22 when |F22| > FLT_EPSILON
__device__ void fm_denormalise(const double (&F0)[3][3], const double* c, const double* sc, double* out) {
    const double T1[3][3] = {{sc[0], 0.0, -sc[0] * c[0]}, {0.0, sc[0], -sc[0] * c[1]}, {0.0, 0.0, 1.0}};
    const double T2[3][3] = {{sc[1], 0.0, -sc[1] * c[2]}, {0.0, sc[1], -sc[1] * c[3]}, {0.0, 0.0, 1.0}};
    double TF[3][3], F[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) TF[i][j] = T2[0][i] * F0[0][j] + T2[1][i] * F0[1][j] + T2[2][i] * F0[2][j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) F[i][j] = TF[i][0] * T1[0][j] + TF[i][1] * T1[1][j] + TF[i][2] * T1[2][j];
    const double f = fabs(F[2][2]) > 1.1920928955078125e-07 ? 1.0 / F[2][2] : 1.0;
    for (int k = 0; k < 9; ++k) out[k] = F[k / 3][k % 3] * f;
}

// cv::solveCubic for c0 x^3 + c1 x^2 + c2 x + c3, c0 != 0: the real roots in its order (trigonometric case: the
// smallest, the largest, the middle one)
__device__ int fm_solve_cubic(const double* c, double* x) {
    const double a1 = c[1] / c[0], a2 = c[2] / c[0], a3 = c[3] / c[0];
    const double Q = (a1 * a1 - 3 * a2) * (1. / 9);
    const double R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1. / 54);
    const double Qcubed = Q * Q * Q;
    const double d = Qcubed - R * R;
    if (d > 0) {
        const double theta = acos(R / sqrt(Qcubed));
        const double t0 = -2 * sqrt(Q), t1 = theta * (1. / 3), t2 = a1 * (1. / 3);
        const double pi = 3.141592653589793;
        x[0] = t0 * cos(t1) - t2;
        x[1] = t0 * cos(t1 + (2. * pi / 3)) - t2;
        x[2] = t0 * cos(t1 - (2. * pi / 3)) - t2;
        return 3;
    }
    double e = cbrt(sqrt(-d) + fabs(R));
    if (R > 0) e = -e;
    x[0] = (e + Q / e) - a1 * (1. / 3);
    return 1;
}

// run7Point on lane 0: the 7 x 9 system's null space in the basis OpenCV's SVD completes it with (two sign vectors of
// cv::RNG(0x12345678) scaled by 1/9, each orthogonalised twice against the row space and the one before it), then the cubic
// det(l f1 + (1 - l) f2) = 0 and one F per real root.  Returns the candidate count (0: no model).
__device__ int fm_seven_point(const double* __restrict__ pts1, const double* __restrict__ pts2, const double* c, const double* sc,
                              double* __restrict__ Fout) {
    __shared__ double q[9][9];    // rows 0..6: an orthonormal basis of the row space; rows 7, 8: f1, f2
    for (int i = 0; i < 7; ++i) {
        double x1, y1, x2, y2, r[9];
        fm_load(pts1, pts2, i, x1, y1, x2, y2);
        fm_row(x1, y1, x2, y2, c, sc, r);
        for (int k = 0; k < 9; ++k) q[i][k] = r[k];
    }
    uint64_t state = 0x12345678ull;
    for (int i = 0; i < 9; ++i) {
        if (i >= 7)
            for (int k = 0; k < 9; ++k) {
                state = (uint64_t)(uint32_t)state * 4164903690ull + (state >> 32);
                q[i][k] = ((uint32_t)state & 256u) ? 1.0 / 9 : -1.0 / 9;
            }
        // Gram-Schmidt, twice, against the rows before it
        for (int pass = 0; pass < 2; ++pass)
            for (int j = 0; j < i; ++j) {
                double d = 0.0;
                for (int k = 0; k < 9; ++k) d += q[i][k] * q[j][k];
                for (int k = 0; k < 9; ++k) q[i][k] -= d * q[j][k];
            }
        double n = 0.0;
        for (int k = 0; k < 9; ++k) n += q[i][k] * q[i][k];
        const double inv = n > 0.0 ? 1.0 / sqrt(n) : 0.0;
        for (int k = 0; k < 9; ++k) q[i][k] *= inv;
    }
    double f1[9], f2[9];
    for (int k = 0; k < 9; ++k) { f2[k] = q[8][k]; f1[k] = q[7][k] - f2[k]; }
    double cf[4];
    {
        double t0 = f2[4] * f2[8] - f2[5] * f2[7], t1 = f2[3] * f2[8] - f2[5] * f2[6], t2 = f2[3] * f2[7] - f2[4] * f2[6];
        cf[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
        cf[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
                f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) -
                f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) + f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
        t0 = f1[4] * f1[8] - f1[5] * f1[7]; t1 = f1[3] * f1[8] - f1[5] * f1[6]; t2 = f1[3] * f1[7] - f1[4] * f1[6];
        cf[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
                f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) -
                f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) + f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
        cf[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
    }
    if (cf[0] == 0.0) return 0;
    double roots[3];
    const int n = fm_solve_cubic(cf, roots);
    for (int k = 0; k < n; ++k) {
        double lambda = roots[k], mu = 1.0;
        const double s = f1[8] * roots[k] + f2[8];
        double F0[3][3];
        if (fabs(s) > 2.220446049250313e-16) {
            mu = 1.0 / s;
            lambda *= mu;
            F0[2][2] = 1.0;
        } else {
            F0[2][2] = 0.0;
        }
        for (int i = 0; i < 8; ++i) F0[i / 3][i % 3] = f1[i] * lambda + f2[i] * mu;
        fm_denormalise(F0, c, sc, Fout + 9 * k);
    }
    return n;
}

// the dense tail, one warp: statuses, run8Point's eigenvector and rank-2 step, or run7Point; fills the record
__global__ void __launch_bounds__(32) fm_solve_kernel(const double* __restrict__ pts1, const double* __restrict__ pts2,
                                                      const int* __restrict__ N_dev, FmWs w, int grid, rf_pose_record_t* __restrict__ rec) {
    __shared__ double s_st[FM_STATS];
    const int N = *N_dev, lane = threadIdx.x;
    if (lane == 0) {
        rec->n_points = N;
        rec->niters = 0;
        rec->best_iter = rec->best_cand = -1;
        rec->ransac_count = -1;
        rec->n_E = 0;
        rec->pose_count = 0;
        rec->pose_cand = rec->pose_index = -1;
        for (int k = 0; k < 4 * ESS_MAXSOL; ++k) rec->pose_counts[k] = 0;
        rec->status = N < 5 ? RF_POSE_TOO_FEW : RF_POSE_NO_MODEL;
    }
    if (N < 7) return;
    fm_stats(w, N, grid, s_st);
    __syncwarp();
    const double* c = s_st;
    const double* sc = s_st + 4;
    if (sc[0] == 0.0 || sc[1] == 0.0) return;                      // a mean distance below FLT_EPSILON
    if (N == 7) {
        if (lane == 0) {
            const int n = fm_seven_point(pts1, pts2, c, sc, rec->E);
            rec->n_E = n;
            rec->status = n > 0 ? RF_POSE_OK : RF_POSE_NO_MODEL;
        }
        return;
    }
    // lane j < 9: column j of A (= row j), column j of V = e_j
    double a[9], v[9], lam;
#pragma unroll
    for (int r = 0; r < 9; ++r) {
        const int i = min(lane, r), k = max(lane, r);
        a[r] = lane < 9 ? s_st[6 + i * 9 - i * (i - 1) / 2 + (k - i)] : 0.0;
        v[r] = r == lane ? 1.0 : 0.0;
    }
    fm_eigen9(a, v, lam);
    // cv::eigen's descending order; the first eight must all be at least DBL_EPSILON in magnitude
    double l[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) l[j] = __shfl_sync(0xffffffffu, lam, j);
    int order[9] = {0, 1, 2, 3, 4, 5, 6, 7, 8};
    for (int i = 0; i < 9; ++i)
        for (int j = i + 1; j < 9; ++j)
            if (l[order[j]] > l[order[i]]) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
    bool degenerate = false;
    for (int i = 0; i < 8; ++i) degenerate |= fabs(l[order[i]]) < 2.220446049250313e-16;
    const int smallest = order[8];
    double f0[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) f0[r] = __shfl_sync(0xffffffffu, v[r], smallest);
    if (lane != 0 || degenerate) return;
    // rank 2: F0 = U diag(w0, w1, 0) V^T from its 3 x 3 SVD
    double A3[3][3], V3[3][3], F0[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A3[i][j] = f0[3 * i + j];
    jacobi_svd<3>(A3, V3);
    double sg[3];
    for (int j = 0; j < 3; ++j) sg[j] = A3[0][j] * A3[0][j] + A3[1][j] * A3[1][j] + A3[2][j] * A3[2][j];
    const int drop = (sg[0] <= sg[1] && sg[0] <= sg[2]) ? 0 : (sg[1] <= sg[2] ? 1 : 2);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double x = 0.0;
            for (int k = 0; k < 3; ++k)
                if (k != drop) x += A3[i][k] * V3[j][k];
            F0[i][j] = x;
        }
    fm_denormalise(F0, c, sc, rec->E);
    rec->n_E = 1;
    rec->status = RF_POSE_OK;
}

}  // namespace rf

using namespace rf;

// ------------------------------------------------------------------------------------------------------------ C ABI
extern "C" size_t rf_yfcc_matches_workspace(int H, int W) {
    const long long P = (long long)(H > 0 ? H : 0) * (W > 0 ? W : 0);
    return align256((size_t)((P + MATCH_TILE - 1) / MATCH_TILE + 1) * sizeof(int));
}

extern "C" int rf_yfcc_matches(const float* flow, const uint8_t* mask, int H, int W, int k, int wB, int hB, int wA, int hA,
                               const double* norm1_host, const double* norm2_host, double* pts1_out, double* pts2_out, int* N_out,
                               void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(H >= 0 && W >= 0 && wB >= 0 && hB >= 0, "rf_yfcc_matches: bad sizes");
    k = ((k % 4) + 4) % 4;
    RF_REQUIRE((k % 2 == 0) ? (H == hB && W == wB) : (H == wB && W == hB), "rf_yfcc_matches: mask shape differs from the rotated grid");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_yfcc_matches_workspace(H, W), "rf_yfcc_matches: workspace too small");
    cudaStream_t st = as_stream(stream);
    const long long P = (long long)H * W;
    const int ntiles = (int)((P + MATCH_TILE - 1) / MATCH_TILE);
    int* tiles = static_cast<int*>(ws);
    if (ntiles == 0) {
        RF_CUDA(cudaMemsetAsync(N_out, 0, sizeof(int), st));
        return 0;
    }
    match_count_kernel<<<ntiles, 256, 0, st>>>(mask, P, tiles);
    RF_LAUNCHED();
    match_scan_kernel<<<1, 1024, 0, st>>>(tiles, ntiles, N_out);
    RF_LAUNCHED();
    const double4 n1 = make_double4(norm1_host[0], norm1_host[1], norm1_host[2], norm1_host[3]);
    const double4 n2 = make_double4(norm2_host[0], norm2_host[1], norm2_host[2], norm2_host[3]);
    match_write_kernel<<<ntiles, 256, 0, st>>>(flow, mask, H, W, k, wB, hB, (float)(wA - 1), (float)(hA - 1), n1, n2, tiles,
                                               pts1_out, pts2_out);
    RF_LAUNCHED();
    return 0;
}

namespace {
struct EssWs {
    int* idx;
    double* candE;
    int* ncand;
    int* counts;
};
EssWs ess_carve(void* ws) {
    unsigned char* p = static_cast<unsigned char*>(ws);
    EssWs w;
    w.idx = reinterpret_cast<int*>(p);
    p += align256((size_t)ESS_ITERS * 5 * sizeof(int));
    w.candE = reinterpret_cast<double*>(p);
    p += align256((size_t)ESS_ITERS * ESS_MAXSOL * 9 * sizeof(double));
    w.ncand = reinterpret_cast<int*>(p);
    p += align256((size_t)ESS_ITERS * sizeof(int));
    w.counts = reinterpret_cast<int*>(p);
    return w;
}
}  // namespace

extern "C" size_t rf_essential_ransac_workspace(int capacity) {
    (void)capacity;
    return align256((size_t)ESS_ITERS * 5 * sizeof(int)) + align256((size_t)ESS_ITERS * ESS_MAXSOL * 9 * sizeof(double)) +
           align256((size_t)ESS_ITERS * sizeof(int)) + align256((size_t)ESS_ITERS * ESS_MAXSOL * sizeof(int));
}

extern "C" int rf_essential_ransac(const double* pts1, const double* pts2, int capacity, const int* N_dev, double threshold,
                                   rf_pose_record_t* rec, uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(capacity >= 0 && N_dev != nullptr && rec != nullptr, "rf_essential_ransac: bad arguments");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_essential_ransac_workspace(capacity), "rf_essential_ransac: workspace too small");
    cudaStream_t st = as_stream(stream);
    EssWs w = ess_carve(ws);
    const float thr2 = (float)(threshold * threshold);
    RF_CUDA(cudaMemsetAsync(w.counts, 0, (size_t)ESS_ITERS * ESS_MAXSOL * sizeof(int), st));
    ess_init_kernel<<<1, 1, 0, st>>>(N_dev, w.idx, rec);
    RF_LAUNCHED();
    ess_solve_kernel<<<(ESS_ITERS + 63) / 64, 64, 0, st>>>(pts1, pts2, N_dev, w.idx, w.candE, w.ncand, ESS_ITERS);
    RF_LAUNCHED();
    const int pts_per_cta = SCORE_THREADS * SCORE_PPT;
    const int grid = capacity > 0 ? (capacity + pts_per_cta - 1) / pts_per_cta : 1;
    const size_t smem = (size_t)ESS_BLOCK * ESS_MAXSOL * 9 * sizeof(double);
    RF_CUDA(cudaFuncSetAttribute(ess_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int b = 0; b < ESS_NBLOCKS; ++b) {
        ess_score_kernel<<<grid, SCORE_THREADS, smem, st>>>(pts1, pts2, N_dev, 0, b * ESS_BLOCK, w.candE, w.ncand, 0, w.counts,
                                                            nullptr, rec, thr2);
        RF_LAUNCHED();
        ess_replay_kernel<<<1, 1, 0, st>>>(b * ESS_BLOCK, w.ncand, w.counts, rec);
        RF_LAUNCHED();
    }
    ess_final_kernel<<<capacity > 0 ? (capacity + 255) / 256 : 1, 256, 0, st>>>(pts1, pts2, capacity, w.candE, w.ncand, rec, thr2,
                                                                                mask_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_essential_samples(const int* N_dev, int* idx_out, void* stream) {
    RF_REQUIRE(N_dev != nullptr && idx_out != nullptr, "rf_essential_samples: bad arguments");
    ess_init_kernel<<<1, 1, 0, as_stream(stream)>>>(N_dev, idx_out, nullptr);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_essential_five_point(const double* pts1, const double* pts2, const int* idx, int nsamples, double* E_out,
                                       int* nsol_out, void* stream) {
    RF_REQUIRE(nsamples >= 0, "rf_essential_five_point: bad sizes");
    if (nsamples == 0) return 0;
    ess_solve_kernel<<<(nsamples + 63) / 64, 64, 0, as_stream(stream)>>>(pts1, pts2, nullptr, idx, E_out, nsol_out, nsamples);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_essential_score(const double* pts1, const double* pts2, int N, const double* E, int nmodels, double threshold,
                                  int* counts_out, float* err_out, void* stream) {
    RF_REQUIRE(N >= 0 && nmodels >= 0 && nmodels <= ESS_BLOCK * ESS_MAXSOL, "rf_essential_score: bad sizes");
    cudaStream_t st = as_stream(stream);
    if (nmodels == 0) return 0;
    RF_CUDA(cudaMemsetAsync(counts_out, 0, (size_t)nmodels * sizeof(int), st));
    if (N == 0) return 0;
    const int pts_per_cta = SCORE_THREADS * SCORE_PPT;
    const size_t smem = (size_t)ESS_BLOCK * ESS_MAXSOL * 9 * sizeof(double);
    RF_CUDA(cudaFuncSetAttribute(ess_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ess_score_kernel<<<(N + pts_per_cta - 1) / pts_per_cta, SCORE_THREADS, smem, st>>>(pts1, pts2, nullptr, N, -1, E, nullptr, nmodels,
                                                                                      counts_out, err_out, nullptr,
                                                                                      (float)(threshold * threshold));
    RF_LAUNCHED();
    return 0;
}

extern "C" size_t rf_recover_pose_workspace(int capacity) {
    const size_t n = (size_t)(capacity > 0 ? capacity : 1);
    return align256(n * sizeof(unsigned long long)) + align256(n);
}

extern "C" int rf_recover_pose(const double* pts1, const double* pts2, int capacity, const uint8_t* mask_in, rf_pose_record_t* rec,
                               uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(capacity >= 0 && rec != nullptr && mask_in != nullptr && mask_out != nullptr, "rf_recover_pose: bad arguments");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_recover_pose_workspace(capacity), "rf_recover_pose: workspace too small");
    cudaStream_t st = as_stream(stream);
    unsigned long long* bits = static_cast<unsigned long long*>(ws);
    uint8_t* chain = static_cast<uint8_t*>(ws) + align256((size_t)(capacity > 0 ? capacity : 1) * sizeof(unsigned long long));
    const int grid = capacity > 0 ? (capacity + 255) / 256 : 1;
    pose_decompose_kernel<<<1, 32, 0, st>>>(rec);
    RF_LAUNCHED();
    pose_cheirality_kernel<<<grid, 256, 0, st>>>(pts1, pts2, capacity, mask_in, rec, bits);
    RF_LAUNCHED();
    pose_select_kernel<<<1, 256, 0, st>>>(mask_in, capacity, rec, bits, chain, mask_out);
    RF_LAUNCHED();
    pose_mask_kernel<<<grid, 256, 0, st>>>(mask_in, capacity, rec, bits, mask_out);
    RF_LAUNCHED();
    return 0;
}

extern "C" size_t rf_fundamental_8point_workspace(int capacity) {
    const size_t g = (size_t)fm_grid(capacity);
    return align256(g * 4 * sizeof(double)) + align256(g * 2 * sizeof(double)) + align256(g * 45 * sizeof(double));
}

// the three reduction passes; CTAs past N exit at once
static void fm_passes(const double* pts1, const double* pts2, const int* N_dev, const FmWs& w, int grid, uint8_t* mask_out,
                      cudaStream_t st) {
    fm_centroid_kernel<<<grid, FM_THREADS, 0, st>>>(pts1, pts2, N_dev, w, mask_out);
    fm_distance_kernel<<<grid, FM_THREADS, 0, st>>>(pts1, pts2, N_dev, w);
    fm_moment_kernel<<<grid, FM_THREADS, 0, st>>>(pts1, pts2, N_dev, w);
}

extern "C" int rf_fundamental_8point(const double* pts1, const double* pts2, int capacity, const int* N_dev, rf_pose_record_t* rec,
                                     uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream) {
    RF_REQUIRE(capacity >= 0 && N_dev != nullptr && rec != nullptr && mask_out != nullptr, "rf_fundamental_8point: bad arguments");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_fundamental_8point_workspace(capacity), "rf_fundamental_8point: workspace too small");
    cudaStream_t st = as_stream(stream);
    const int grid = fm_grid(capacity);
    const FmWs w = fm_carve(ws, grid);
    fm_passes(pts1, pts2, N_dev, w, grid, mask_out, st);
    RF_LAUNCHED();
    fm_solve_kernel<<<1, 32, 0, st>>>(pts1, pts2, N_dev, w, grid, rec);
    RF_LAUNCHED();
    return 0;
}

extern "C" int rf_fundamental_moments(const double* pts1, const double* pts2, int capacity, const int* N_dev, double* out, void* ws,
                                      size_t ws_bytes, void* stream) {
    RF_REQUIRE(capacity >= 0 && N_dev != nullptr && out != nullptr, "rf_fundamental_moments: bad arguments");
    RF_REQUIRE(ws != nullptr && ws_bytes >= rf_fundamental_8point_workspace(capacity), "rf_fundamental_moments: workspace too small");
    cudaStream_t st = as_stream(stream);
    const int grid = fm_grid(capacity);
    const FmWs w = fm_carve(ws, grid);
    fm_passes(pts1, pts2, N_dev, w, grid, nullptr, st);
    RF_LAUNCHED();
    fm_stats_kernel<<<1, 32, 0, st>>>(N_dev, w, grid, out);
    RF_LAUNCHED();
    return 0;
}
