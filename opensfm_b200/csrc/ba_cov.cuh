// Rig-instance pose covariances of bundle adjustment (Ceres Covariance on the reference's
// BundleAdjuster::ComputeCovariances, bundle_adjuster.cc:1123-1194), dense fp64 on the tensor cores.
//
// The marginal covariance of the camera-side parameters is S^-1, S the undamped, Jacobi-scaled reduced
// camera system at the final parameters.  S (n_c x n_c) is expanded into a dense column-major matrix whose
// columns are permuted so that the m = 6 * (#free rig instances) instance columns come last.  With
// S = L L^T and L = [L11 0; L21 L22], the trailing block of S^-1 is L22^-T L22^-1: only L22 (m x m) has
// to be inverted, the leading columns never enter a solve.
//   cov_densify       block-sparse S -> dense lower triangle (+ original diagonal for the pivot test)
//   cov_potrf_diag    Cholesky of one diagonal block (pivot test) + the inverse of its factor
//   cov_gemm<TRSM>    panel: L21 = A21 L11^-T
//   cov_gemm<SYRK>    trailing update A22 -= L21 L21^T (lower tiles)
//   cov_gemm<TRI_*>   X = L22^-1, blocked right-looking, the diagonal-block inverses of the Cholesky reused
//   cov_blocks        C_i = diag(s) X_i^T X_i diag(s) per free instance (X_i its 6 columns of X)
// The panel and trailing products run on mma.sync.m8n8k4.f64 (dmma884, ba_reduced.cuh).
//
// Rank: J counts as rank deficient when a Cholesky pivot is <= COV_TAU times the original diagonal entry,
// on every point's scaled 3x3 V (ba_point_blocks / ba_schur, point_rank_deficient) or on S.
//
// Included by ba.cu after ba_reduced.cuh.
#pragma once

namespace osfm {

constexpr int COV_NB = 64;                 // panel width = output tile of cov_gemm
constexpr int COV_LDS = COV_NB + 4;        // shared-memory row pitch: a fragment load hits each bank pair at most twice
constexpr int COV_THREADS = 256;
// device flags, read once by the host after the last kernel (COV_F_POINT_RANK: ba_point_blocks / ba_schur)
enum { COV_F_CHOL = 1, COV_F_CHOL_COL = 2, COV_F_NONFINITE = 3, COV_F_COUNT = 4 };

// One warp per stored upper block: scatter into the permuted dense lower triangle, column-major (ld = nc).
__global__ void __launch_bounds__(256)
    cov_densify(const int4* __restrict__ upper, int n_upper, BsrView h, const double* __restrict__ Sval,
                const int* __restrict__ perm, int nc, double* __restrict__ A, double* __restrict__ d0) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_upper) return;
  const int4 u = upper[w];
  const int szi = h.blk_sz[u.x], szj = h.blk_sz[u.y], oi = h.blk_off[u.x], oj = h.blk_off[u.y];
  for (int e = lane; e < szi * szj; e += 32) {
    const int r = e / szj, c = e % szj;
    if (u.x == u.y && c < r) continue;   // diagonal blocks: upper triangle only
    const int gi = perm[oi + r], gj = perm[oj + c];
    const double val = Sval[u.z + e];
    A[(size_t)max(gi, gj) + (size_t)min(gi, gj) * nc] = val;
    if (gi == gj) d0[gi] = val;
  }
}

// Cholesky of the kb x kb diagonal block at (k0, k0) in shared memory with the pivot test, then W = L11^-1
// (lower, column-major, ld COV_NB) for the panel solve and the triangular inverse.
__global__ void __launch_bounds__(COV_THREADS, 1)
    cov_potrf_diag(double* __restrict__ A, int n, int k0, int kb, const double* __restrict__ d0, double* __restrict__ W,
                   int* __restrict__ flags) {
  if (flags[COV_F_CHOL]) return;
  extern __shared__ double cs[];
  double* a = cs;                          // [COV_NB][COV_NB + 1], a[i * (COV_NB + 1) + j] = L(i, j)
  double* x = cs + COV_NB * (COV_NB + 1);  // the same for W
  constexpr int LD = COV_NB + 1;
  __shared__ int fail;
  const int tid = threadIdx.x;
  if (tid == 0) fail = 0;
  for (int e = tid; e < kb * kb; e += COV_THREADS) {
    const int i = e % kb, j = e / kb;
    a[i * LD + j] = i >= j ? A[(size_t)(k0 + i) + (size_t)(k0 + j) * n] : 0.0;
  }
  __syncthreads();
  for (int j = 0; j < kb; ++j) {
    if (tid == 0) {
      const double p = a[j * LD + j];
      if (!(p > COV_TAU * d0[k0 + j])) {
        fail = 1;
        flags[COV_F_CHOL_COL] = k0 + j;
        flags[COV_F_CHOL] = 1;
      } else {
        a[j * LD + j] = sqrt(p);
      }
    }
    __syncthreads();
    if (fail) return;
    const double ljj = a[j * LD + j];
    for (int i = j + 1 + tid; i < kb; i += COV_THREADS) a[i * LD + j] /= ljj;
    __syncthreads();
    const int t = kb - j - 1;   // trailing lower triangle, t x t
    for (int e = tid; e < t * t; e += COV_THREADS) {
      const int i = j + 1 + e / t, c = j + 1 + e % t;
      if (c <= i) a[i * LD + c] -= a[i * LD + j] * a[c * LD + j];
    }
    __syncthreads();
  }
  for (int e = tid; e < kb * kb; e += COV_THREADS) {
    const int i = e % kb, j = e / kb;
    if (i >= j) A[(size_t)(k0 + i) + (size_t)(k0 + j) * n] = a[i * LD + j];
  }
  // W = L^-1 by forward substitution, one column per thread
  if (tid < kb) {
    const int j = tid;
    for (int i = 0; i < j; ++i) x[i * LD + j] = 0.0;
    x[j * LD + j] = 1.0 / a[j * LD + j];
    for (int i = j + 1; i < kb; ++i) {
      double s = 0.0;
      for (int t = j; t < i; ++t) s += a[i * LD + t] * x[t * LD + j];
      x[i * LD + j] = -s / a[i * LD + i];
    }
  }
  __syncthreads();
  for (int e = tid; e < COV_NB * COV_NB; e += COV_THREADS) {
    const int i = e % COV_NB, j = e / COV_NB;
    W[e] = (i < kb && j < kb) ? x[i * LD + j] : 0.0;
  }
}

enum { COV_TRSM = 0, COV_SYRK = 1, COV_TRI_DIAG = 2, COV_TRI_UPD = 3 };
struct CovGemm {
  double* A;          // dense S / L, column-major, ld n
  int n;
  double* X;          // L22^-1, column-major, ld m
  int m, n1;          // L22 = A[n1:, n1:]
  const double* W;    // inverse of the current diagonal block (ld COV_NB)
  int k0, kb;         // current block: columns [k0, k0 + kb) of A (TRSM, SYRK) or of L22 (TRI_*)
  const int* flags;
};

// One 64 x 64 output tile per CTA: C(i, j) = sum_t P(i, t) Q(j, t), t < kb, with P and Q staged as [row][t]
// in shared memory.  Warp w owns the eight 8x8 tiles of rows [8w, 8w + 8).
//   TRSM     A21 tile rows r (below the block) := A21 W^T                  grid (row tiles, 1)
//   SYRK     A22(r, c) -= L21(r) . L21(c), lower tiles only                grid (row tiles, col tiles)
//   TRI_DIAG X(k rows, c) := W X(k rows, c)                                grid (1, col tiles of [0, k0 + kb))
//   TRI_UPD  X(r, c) -= L22(r, k cols) X(k rows, c), r >= k0 + kb           grid (row tiles, col tiles)
template <int MODE>
__global__ void __launch_bounds__(COV_THREADS)
    cov_gemm(CovGemm g) {
  if (g.flags[COV_F_CHOL]) return;
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (MODE == COV_SYRK && tj > ti) return;
  extern __shared__ double cs[];
  double* P = cs;
  double* Q = cs + COV_NB * COV_LDS;
  const int kb = g.kb, kbp = (kb + 3) & ~3;
  const int tid = threadIdx.x;
  // rows of P / Q (global indices in their matrices) and their counts
  int pr0, np, qr0, nq;
  if (MODE == COV_TRSM || MODE == COV_SYRK) {
    const int s = g.k0 + kb;
    pr0 = s + ti * COV_NB; np = min(COV_NB, g.n - pr0);
    qr0 = MODE == COV_TRSM ? 0 : s + tj * COV_NB;
    nq = MODE == COV_TRSM ? kb : min(COV_NB, g.n - qr0);
  } else if (MODE == COV_TRI_DIAG) {
    pr0 = 0; np = kb;
    qr0 = tj * COV_NB; nq = min(COV_NB, g.k0 + kb - qr0);
  } else {
    pr0 = g.k0 + kb + ti * COV_NB; np = min(COV_NB, g.m - pr0);
    qr0 = tj * COV_NB; nq = min(COV_NB, g.k0 + kb - qr0);
  }
  // P: consecutive threads walk rows (contiguous in the column-major sources)
  for (int e = tid; e < COV_NB * kbp; e += COV_THREADS) {
    const int i = e % COV_NB, t = e / COV_NB;
    double v = 0.0;
    if (i < np && t < kb) {
      if (MODE == COV_TRSM || MODE == COV_SYRK) v = g.A[(size_t)(pr0 + i) + (size_t)(g.k0 + t) * g.n];
      else if (MODE == COV_TRI_DIAG) v = g.W[i + t * COV_NB];
      else v = g.A[(size_t)(g.n1 + pr0 + i) + (size_t)(g.n1 + g.k0 + t) * g.n];
    }
    P[i * COV_LDS + t] = v;
  }
  if (MODE == COV_TRSM || MODE == COV_SYRK) {
    for (int e = tid; e < COV_NB * kbp; e += COV_THREADS) {
      const int j = e % COV_NB, t = e / COV_NB;
      double v = 0.0;
      if (j < nq && t < kb) v = MODE == COV_TRSM ? g.W[j + t * COV_NB] : g.A[(size_t)(qr0 + j) + (size_t)(g.k0 + t) * g.n];
      Q[j * COV_LDS + t] = v;
    }
  } else {   // Q(j, t) = X(k0 + t, qr0 + j): consecutive threads walk t
    for (int e = tid; e < COV_NB * kbp; e += COV_THREADS) {
      const int t = e % kbp, j = e / kbp;
      Q[j * COV_LDS + t] = (j < nq && t < kb) ? g.X[(size_t)(g.k0 + t) + (size_t)(qr0 + j) * g.m] : 0.0;
    }
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[8][2];
#pragma unroll
  for (int jt = 0; jt < 8; ++jt) acc[jt][0] = acc[jt][1] = 0.0;
  const double* pa = P + (warp * 8 + fr) * COV_LDS + fk;
  for (int k = 0; k < kbp; k += 4) {
    const double av = pa[k];
#pragma unroll
    for (int jt = 0; jt < 8; ++jt) dmma884(acc[jt][0], acc[jt][1], av, Q[(jt * 8 + fr) * COV_LDS + k + fk]);
  }
  // TRSM / TRI_DIAG overwrite the rows they read: every CTA has staged its operands before anyone writes
  const int i = warp * 8 + fr;
#pragma unroll
  for (int jt = 0; jt < 8; ++jt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = jt * 8 + 2 * fk + h;
      if (i >= np || j >= nq) continue;
      const double v = acc[jt][h];
      if (MODE == COV_TRSM) {
        g.A[(size_t)(pr0 + i) + (size_t)(g.k0 + j) * g.n] = v;
      } else if (MODE == COV_SYRK) {
        if (pr0 + i >= qr0 + j) g.A[(size_t)(pr0 + i) + (size_t)(qr0 + j) * g.n] -= v;
      } else if (MODE == COV_TRI_DIAG) {
        g.X[(size_t)(g.k0 + i) + (size_t)(qr0 + j) * g.m] = v;
      } else {
        g.X[(size_t)(pr0 + i) + (size_t)(qr0 + j) * g.m] -= v;
      }
    }
}

__global__ void cov_identity(double* X, int m) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < (long long)m * m) X[e] = (e % m == e / m) ? 1.0 : 0.0;
}

// One CTA per free instance q (columns [6q, 6q + 6) of X = L22^-1, rows >= 6q):
// C = diag(s) X_q^T X_q diag(s), written row-major into out[inst * 36].
__global__ void __launch_bounds__(COV_THREADS)
    cov_blocks(const double* __restrict__ X, int m, const int* __restrict__ inst_of, const int* __restrict__ inst_poff,
               const double* __restrict__ scale, const int* __restrict__ flags, double* __restrict__ out,
               int* __restrict__ out_flags) {
  if (flags[COV_F_CHOL]) return;
  const int q = blockIdx.x, c0 = 6 * q, tid = threadIdx.x;
  double acc[21];
#pragma unroll
  for (int e = 0; e < 21; ++e) acc[e] = 0.0;
  for (int r = c0 + tid; r < m; r += COV_THREADS) {
    double x[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) x[a] = X[(size_t)r + (size_t)(c0 + a) * m];
    int e = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = a; b < 6; ++b) acc[e++] += x[a] * x[b];
  }
  __shared__ double red[COV_THREADS / 32][21];
#pragma unroll
  for (int e = 0; e < 21; ++e) {
    double v = acc[e];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) red[tid >> 5][e] = v;
  }
  __syncthreads();
  if (tid < 21) {
    double v = 0.0;
    for (int w = 0; w < COV_THREADS / 32; ++w) v += red[w][tid];
    int a = 0, e = tid;
    while (e >= 6 - a) { e -= 6 - a; ++a; }
    const int b = a + e;
    const int inst = inst_of[q], g0 = inst_poff[inst];
    v *= scale[g0 + a] * scale[g0 + b];
    out[(size_t)inst * 36 + a * 6 + b] = v;
    out[(size_t)inst * 36 + b * 6 + a] = v;
    if (!isfinite(v)) out_flags[COV_F_NONFINITE] = 1;
  }
}

}  // namespace osfm
