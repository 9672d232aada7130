// Hierarchy-based class embeddings (compute_class_embedding.py): the LCS-height distance table, a blocked fp64 Cholesky
// factorisation, one-sided block Jacobi on the columns of a matrix, the embeddings' self-check, and the small fp64 steps
// between them.  Everything is float64; the O(n^3) parts (the Cholesky trailing update, the Jacobi Gram matrices and
// rotations) run on fp64 tensor-core tiles (mma.sync m8n8k4 .f64, "DMMA").  No float atomics: reruns give the same bits.
//
//   unitsphere  = L,                 S = 1 - D = L L^T
//   spheres     = [0; L],            G_ij = (D_0i^2 + D_0j^2 - D_ij^2) / 2 = L L^T   (i, j >= 1)
//   approx_sim  = L J,               J orthogonal with the columns of L J mutually orthogonal: (L J)(L J)^T = S, so the
//                                    squared column norms are the eigenvalues of S and L J = Q sqrt(Lambda)
//   mds         = (X - mean) J,      X the spheres embedding; (X - mean)(X - mean)^T = -1/2 H D^2 H
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace se {

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

// ------------------------------------------------------------------------------------------------ LCS-height table
// One pair per thread.  A class's list holds its ancestors (itself included) as ranks in the order (-depth, node index),
// so the first common entry of two ascending lists is the deepest common subsumer with ClassHierarchy._lcs_ix's tie rule.
constexpr int LCS_TILE = 16;
constexpr int LCS_MAXLEN = 64;

__global__ void __launch_bounds__(LCS_TILE * LCS_TILE)
lcs_height_kernel(const int* __restrict__ off, const int* __restrict__ anc, const int* __restrict__ height, int max_height,
                  int C, double* __restrict__ D, long long ldd) {
  pdl_grid_sync();
  __shared__ int rows[LCS_TILE][LCS_MAXLEN], cols[LCS_TILE][LCS_MAXLEN];
  __shared__ int rlen[LCS_TILE], clen[LCS_TILE];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int i0 = blockIdx.y * LCS_TILE, j0 = blockIdx.x * LCS_TILE;
  const int tid = ty * LCS_TILE + tx;
  if (tid < LCS_TILE) {
    const int c = i0 + tid;
    rlen[tid] = c < C ? off[c + 1] - off[c] : 0;
  } else if (tid < 2 * LCS_TILE) {
    const int c = j0 + tid - LCS_TILE;
    clen[tid - LCS_TILE] = c < C ? off[c + 1] - off[c] : 0;
  }
  __syncthreads();
  for (int e = tid; e < LCS_TILE * LCS_MAXLEN; e += LCS_TILE * LCS_TILE) {
    const int r = e / LCS_MAXLEN, k = e % LCS_MAXLEN;
    if (k < rlen[r]) rows[r][k] = anc[off[i0 + r] + k];
    if (k < clen[r]) cols[r][k] = anc[off[j0 + r] + k];
  }
  __syncthreads();
  const int i = i0 + ty, j = j0 + tx;
  if (i >= C || j >= C) return;
  double d = 0.0;
  if (i != j) {
    const int na = rlen[ty], nb = clen[tx];
    int a = 0, b = 0, h = -1;
    while (a < na && b < nb) {
      const int va = rows[ty][a], vb = cols[tx][b];
      if (va == vb) { h = va; break; }
      if (va < vb) ++a; else ++b;
    }
    d = h < 0 ? __longlong_as_double(0x7ff8000000000000ll) : (double)height[h] / (double)max_height;
  }
  D[(long long)i * ldd + j] = d;
}

// ------------------------------------------------------------------------------------------------ Cholesky
// Right-looking, panels of CH_NB columns: the diagonal block in one CTA (SIMT), the rows below it by substitution
// (SIMT), and the trailing update A22 -= L21 L21^T of the lower triangle on DMMA tiles.
constexpr int CH_NB = 32;
constexpr int CH_TRSM_ROWS = 128;
constexpr int CH_TILE = 64;

__global__ void __launch_bounds__(256) chol_panel_kernel(double* __restrict__ A, long long lda, int n, int k0,
                                                         int* __restrict__ status) {
  pdl_grid_sync();
  __shared__ double T[CH_NB][CH_NB + 1];
  __shared__ double piv;
  const int nb = min(CH_NB, n - k0), tid = threadIdx.x;
  for (int e = tid; e < CH_NB * CH_NB; e += blockDim.x) {
    const int i = e / CH_NB, j = e % CH_NB;
    T[i][j] = (i < nb && j <= i) ? A[(long long)(k0 + i) * lda + k0 + j] : 0.0;
  }
  __syncthreads();
  for (int j = 0; j < nb; ++j) {
    if (tid == 0) {
      const double d = T[j][j];
      if (!(d > 0.0)) {                 // not positive definite (or NaN): report the first such row, keep the raw pivot
        if (*status < 0) *status = k0 + j;
        piv = sqrt(d);
      } else {
        piv = sqrt(d);
        T[j][j] = piv;
      }
    }
    __syncthreads();
    for (int i = j + 1 + tid; i < nb; i += blockDim.x) T[i][j] /= piv;
    __syncthreads();
    const int m = nb - j - 1;
    for (int e = tid; e < m * m; e += blockDim.x) {
      const int i = j + 1 + e / m, k = j + 1 + e % m;
      if (k <= i) T[i][k] -= T[i][j] * T[k][j];
    }
    __syncthreads();
  }
  for (int e = tid; e < nb * nb; e += blockDim.x) {
    const int i = e / nb, j = e % nb;
    A[(long long)(k0 + i) * lda + k0 + j] = j <= i ? T[i][j] : 0.0;
  }
}

// rows k0+nb .. n-1 of the panel: L21 = A21 L11^-T, one row per thread, staged through shared memory
__global__ void __launch_bounds__(CH_TRSM_ROWS) chol_trsm_kernel(double* __restrict__ A, long long lda, int n, int k0) {
  pdl_grid_sync();
  __shared__ double L[CH_NB][CH_NB + 1];
  __shared__ double X[CH_TRSM_ROWS][CH_NB + 1];
  const int nb = min(CH_NB, n - k0), tid = threadIdx.x;
  const int r0 = k0 + nb + blockIdx.x * CH_TRSM_ROWS;
  for (int e = tid; e < CH_NB * CH_NB; e += blockDim.x) {
    const int i = e / CH_NB, j = e % CH_NB;
    L[i][j] = (i < nb && j <= i) ? A[(long long)(k0 + i) * lda + k0 + j] : 0.0;
  }
  for (int e = tid; e < CH_TRSM_ROWS * CH_NB; e += blockDim.x) {
    const int r = e / CH_NB, k = e % CH_NB;
    X[r][k] = (r0 + r < n && k < nb) ? A[(long long)(r0 + r) * lda + k0 + k] : 0.0;
  }
  __syncthreads();
  for (int j = 0; j < nb; ++j) {
    double v = X[tid][j];
    for (int k = 0; k < j; ++k) v -= X[tid][k] * L[j][k];
    X[tid][j] = v / L[j][j];
  }
  __syncthreads();
  for (int e = tid; e < CH_TRSM_ROWS * CH_NB; e += blockDim.x) {
    const int r = e / CH_NB, k = e % CH_NB;
    if (r0 + r < n && k < nb) A[(long long)(r0 + r) * lda + k0 + k] = X[r][k];
  }
}

// A22 -= L21 L21^T on the lower triangle: one 64 x 64 tile per CTA (tiles above the diagonal exit), four warps of
// 32 x 32, the panel's nb <= 32 columns as the reduction
__global__ void __launch_bounds__(128) chol_update_kernel(double* __restrict__ A, long long lda, int n, int k0) {
  pdl_grid_sync();
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj > bi) return;
  __shared__ double Li[CH_TILE][CH_NB + 1], Lj[CH_TILE][CH_NB + 1];
  const int nb = min(CH_NB, n - k0), s = k0 + nb;
  const int r0 = s + bi * CH_TILE, c0 = s + bj * CH_TILE, tid = threadIdx.x;
  for (int e = tid; e < CH_TILE * CH_NB; e += blockDim.x) {
    const int r = e / CH_NB, k = e % CH_NB;
    Li[r][k] = (r0 + r < n && k < nb) ? A[(long long)(r0 + r) * lda + k0 + k] : 0.0;
    Lj[r][k] = (c0 + r < n && k < nb) ? A[(long long)(c0 + r) * lda + k0 + k] : 0.0;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
  double acc[4][4][2] = {};
#pragma unroll
  for (int kk = 0; kk < CH_NB; kk += 4) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = Li[wr + 8 * i + g][kk + t];
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = Lj[wc + 8 * j + g][kk + t];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma(acc[i][j], a[i], b[j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int row = r0 + wr + 8 * i + g, col = c0 + wc + 8 * j + 2 * t + q;
        if (row < n && col <= row) A[(long long)row * lda + col] -= acc[i][j][q];
      }
}

__global__ void zero_upper_kernel(double* __restrict__ A, long long lda, int n) {
  pdl_grid_sync();
  const long long total = (long long)n * n;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / n), j = (int)(e % n);
    if (j > i) A[(long long)i * lda + j] = 0.0;
  }
}

// ------------------------------------------------------------------------------------------------ small fp64 steps
// op 0: out [C, C] = 1 - D;  op 1: out [C-1, C-1] = G_ij = (D_0,i+1^2 + D_0,j+1^2 - D_i+1,j+1^2) / 2
__global__ void class_gram_kernel(const double* __restrict__ D, long long ldd, int C, int op, double* __restrict__ out,
                                  long long ldo) {
  pdl_grid_sync();
  const int n = op == 0 ? C : C - 1;
  const long long total = (long long)n * n;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / n), j = (int)(e % n);
    double v;
    if (op == 0) {
      v = 1.0 - D[(long long)i * ldd + j];
    } else {
      const double a = D[i + 1], b = D[j + 1], d = D[(long long)(i + 1) * ldd + j + 1];
      v = (a * a + b * b - d * d) / 2.0;
    }
    out[(long long)i * ldo + j] = v;
  }
}

// one thread per column, rows in increasing order: op 0 out[j] = sum_i X_ij^2; op 1 X_ij -= mean_i X_ij (in place)
__global__ void column_op_kernel(double* __restrict__ X, long long ldx, int m, int n, int op, double* __restrict__ out) {
  pdl_grid_sync();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double s = 0.0;
  if (op == 0) {
    for (int i = 0; i < m; ++i) { const double v = X[(long long)i * ldx + j]; s += v * v; }
    out[j] = s;
  } else {
    for (int i = 0; i < m; ++i) s += X[(long long)i * ldx + j];
    const double mean = s / m;
    for (int i = 0; i < m; ++i) X[(long long)i * ldx + j] -= mean;
  }
}

__global__ void gather_columns_kernel(const double* __restrict__ X, long long ldx, int m, const int* __restrict__ cols, int k,
                                      double* __restrict__ Y, long long ldy) {
  pdl_grid_sync();
  const long long total = (long long)m * k;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / k), c = (int)(e % k);
    Y[(long long)i * ldy + c] = X[(long long)i * ldx + cols[c]];
  }
}

// one warp per row: x /= ||x||_2
__global__ void row_normalize_kernel(double* __restrict__ X, long long ldx, int m, int n) {
  pdl_grid_sync();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= m) return;
  double* x = X + (long long)row * ldx;
  double s = 0.0;
  for (int j = lane; j < n; j += 32) s += x[j] * x[j];
  const double nrm = sqrt(warp_sum(s));
  for (int j = lane; j < n; j += 32) x[j] /= nrm;
}

// ------------------------------------------------------------------------------------------------ block Jacobi
// Columns in blocks of JB; the blocks meet in round-robin order (block 0 fixed, the others rotating), a round pairing
// every block once.  Per block pair: the 2JB x 2JB Gram matrix of its columns on DMMA, cyclic two-sided Jacobi on it in
// shared memory with the accumulated rotation V (jacobi_gram_kernel), then [X_I X_J] <- [X_I X_J] V on DMMA
// (jacobi_apply_kernel).  A pair (a, b) is rotated only when |a.b| > tol |a| |b| and neither column is zero; a sweep in
// which no Gram matrix has such a pair ends the iteration.  Columns past n (the padding of the last block, and the dummy
// block of an odd block count) read as zero and are never written.
constexpr int JB = 16, JP = 2 * JB;
constexpr int JG_WARPS = 8;
constexpr int JA_ROWS = 64;
constexpr int J_INNER_SWEEPS = 8;

__device__ __forceinline__ int rr_block(int pos, int round, int nbk) { return pos == 0 ? 0 : 1 + (pos - 1 + round) % (nbk - 1); }
__device__ __forceinline__ int pair_col(int c, int bI, int bJ) { return c < JB ? bI * JB + c : bJ * JB + c - JB; }

__global__ void __launch_bounds__(JG_WARPS * 32)
jacobi_gram_kernel(const double* __restrict__ X, long long ldx, int m, int n, int nbk, int round, double tol,
                   double* __restrict__ Vws, int* __restrict__ rotated, int* __restrict__ notconv) {
  pdl_grid_sync();
  __shared__ double G[JP][JP + 1], V[JP][JP + 1];
  __shared__ double cs[JB], sn[JB], tt[JB], al0[JB], be0[JB], ga0[JB];
  __shared__ int P[JB], Q[JB];
  __shared__ int any, any_sweep;
  const int p = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int bI = rr_block(p, round, nbk), bJ = rr_block(nbk - 1 - p, round, nbk);
  int col[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) col[q] = pair_col(8 * q + g, bI, bJ);
  double acc[4][4][2] = {};
  for (int r = 4 * warp + t; r - t < m; r += 4 * JG_WARPS) {
    double v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = (r < m && col[q] < n) ? X[(long long)r * ldx + col[q]] : 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma(acc[i][j], v[i], v[j]);
  }
  // the warps' partial Gram matrices, added in warp order
  for (int w = 0; w < JG_WARPS; ++w) {
    if (warp == w) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            double& d = G[8 * i + g][8 * j + 2 * t + q];
            d = w == 0 ? acc[i][j][q] : d + acc[i][j][q];
          }
    }
    __syncthreads();
  }
  for (int e = tid; e < JP * JP; e += blockDim.x) V[e / JP][e % JP] = (e / JP == e % JP) ? 1.0 : 0.0;
  if (tid == 0) any = 0;
  __syncthreads();
  for (int sweep = 0; sweep < J_INNER_SWEEPS; ++sweep) {
    if (tid == 0) any_sweep = 0;
    __syncthreads();
    for (int step = 0; step < JP - 1; ++step) {
      if (tid < JB) {
        const int a = tid == 0 ? 0 : 1 + (tid - 1 + step) % (JP - 1);
        const int b = 1 + (JP - 2 - tid + step) % (JP - 1);
        const double al = G[a][a], be = G[b][b], ga = G[a][b];
        double c = 1.0, s = 0.0, tn = 0.0;
        if (al > 0.0 && be > 0.0 && fabs(ga) > tol * sqrt(al) * sqrt(be)) {
          const double zeta = (be - al) / (2.0 * ga);
          tn = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
          c = 1.0 / sqrt(1.0 + tn * tn);
          s = c * tn;
          any_sweep = 1;
        }
        P[tid] = a; Q[tid] = b; cs[tid] = c; sn[tid] = s; tt[tid] = tn;
        al0[tid] = al; be0[tid] = be; ga0[tid] = ga;
      }
      __syncthreads();
      for (int e = tid; e < JP * JB; e += blockDim.x) {          // columns: G <- G J, V <- V J
        const int r = e / JB, k = e % JB;
        if (sn[k] != 0.0) {
          const int a = P[k], b = Q[k];
          const double c = cs[k], s = sn[k];
          const double ga = G[r][a], gb = G[r][b], va = V[r][a], vb = V[r][b];
          G[r][a] = c * ga - s * gb; G[r][b] = s * ga + c * gb;
          V[r][a] = c * va - s * vb; V[r][b] = s * va + c * vb;
        }
      }
      __syncthreads();
      for (int e = tid; e < JP * JB; e += blockDim.x) {          // rows: G <- J^T G
        const int r = e / JB, k = e % JB;
        if (sn[k] != 0.0) {
          const int a = P[k], b = Q[k];
          const double c = cs[k], s = sn[k];
          const double ga = G[a][r], gb = G[b][r];
          G[a][r] = c * ga - s * gb; G[b][r] = s * ga + c * gb;
        }
      }
      __syncthreads();
      if (tid < JB && sn[tid] != 0.0) {                          // the rotated pair's 2 x 2 block, exactly diagonal
        const int a = P[tid], b = Q[tid];
        G[a][a] = al0[tid] - tt[tid] * ga0[tid];
        G[b][b] = be0[tid] + tt[tid] * ga0[tid];
        G[a][b] = G[b][a] = 0.0;
      }
      __syncthreads();
    }
    if (any_sweep == 0) break;
    if (tid == 0) any = 1;
    __syncthreads();
  }
  if (any) {
    // V carries the rounding of every rotation it accumulated, and each round applies it to the whole matrix: one
    // Newton-Schulz step V <- V (3I - V^T V) / 2 makes it orthogonal to working precision again, so the column norms
    // (the eigenvalues) do not drift over the thousands of rounds of a large problem.  G is free now and holds V^T V.
    for (int e = tid; e < JP * JP; e += blockDim.x) {
      const int i = e / JP, j = e % JP;
      double s = 0.0;
      for (int k = 0; k < JP; ++k) s = fma(V[k][i], V[k][j], s);
      G[i][j] = (i == j ? 3.0 : 0.0) - s;
    }
    __syncthreads();
    double w[JP * JP / (JG_WARPS * 32)];
    for (int u = 0, e = tid; e < JP * JP; e += blockDim.x, ++u) {
      const int i = e / JP, j = e % JP;
      double s = 0.0;
      for (int k = 0; k < JP; ++k) s = fma(V[i][k], G[k][j], s);
      w[u] = 0.5 * s;
    }
    __syncthreads();
    for (int u = 0, e = tid; e < JP * JP; e += blockDim.x, ++u) V[e / JP][e % JP] = w[u];
    __syncthreads();
  }
  const long long base = (long long)p * JP * JP;
  for (int e = tid; e < JP * JP; e += blockDim.x) Vws[base + e] = V[e / JP][e % JP];
  if (tid == 0) {
    rotated[p] = any;
    if (any) *notconv = 1;
  }
}

__global__ void __launch_bounds__(128)
jacobi_apply_kernel(double* __restrict__ X, long long ldx, int m, int n, int nbk, int round, const double* __restrict__ Vws,
                    const int* __restrict__ rotated) {
  pdl_grid_sync();
  const int p = blockIdx.x;
  if (!rotated[p]) return;
  __shared__ double V[JP][JP + 1], Xs[JA_ROWS][JP + 1];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int bI = rr_block(p, round, nbk), bJ = rr_block(nbk - 1 - p, round, nbk);
  const int r0 = blockIdx.y * JA_ROWS;
  const long long base = (long long)p * JP * JP;
  for (int e = tid; e < JP * JP; e += blockDim.x) V[e / JP][e % JP] = Vws[base + e];
  for (int e = tid; e < JA_ROWS * JP; e += blockDim.x) {
    const int r = e / JP, c = pair_col(e % JP, bI, bJ);
    Xs[r][e % JP] = (r0 + r < m && c < n) ? X[(long long)(r0 + r) * ldx + c] : 0.0;
  }
  __syncthreads();
  const int wr = warp * 16;
  double acc[2][4][2] = {};
#pragma unroll
  for (int kk = 0; kk < JP; kk += 4) {
    double a[2], b[4];
#pragma unroll
    for (int i = 0; i < 2; ++i) a[i] = Xs[wr + 8 * i + g][kk + t];
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = V[kk + t][8 * j + g];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) dmma(acc[i][j], a[i], b[j]);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int row = r0 + wr + 8 * i + g, c = pair_col(8 * j + 2 * t + q, bI, bJ);
        if (row < m && c < n) X[(long long)row * ldx + c] = acc[i][j][q];
      }
}

// ------------------------------------------------------------------------------------------------ self-check
// mode 0: |E_i.E_j - (1 - D_ij)|;  mode 1: |‖E_i - E_j‖ - D_ij|.  64 x 64 pairs per CTA, 4 x 4 per thread, then the
// per-tile max and sum; dev_final_kernel combines the tiles in index order.
constexpr int DV_T = 64, DV_K = 16;

__global__ void __launch_bounds__(256)
deviation_tile_kernel(const double* __restrict__ E, long long lde, int C, int dim, const double* __restrict__ D, long long ldd,
                      int mode, double* __restrict__ ws) {
  pdl_grid_sync();
  __shared__ double Ai[DV_K][DV_T + 1], Aj[DV_K][DV_T + 1];
  __shared__ double rmax[256], rsum[256];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int i0 = blockIdx.y * DV_T, j0 = blockIdx.x * DV_T;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < dim; k0 += DV_K) {
    for (int e = tid; e < DV_T * DV_K; e += 256) {
      const int r = e / DV_K, k = e % DV_K;
      Ai[k][r] = (i0 + r < C && k0 + k < dim) ? E[(long long)(i0 + r) * lde + k0 + k] : 0.0;
      Aj[k][r] = (j0 + r < C && k0 + k < dim) ? E[(long long)(j0 + r) * lde + k0 + k] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < DV_K; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { a[u] = Ai[k][ty + 16 * u]; b[u] = Aj[k][tx + 16 * u]; }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          if (mode == 0) {
            acc[u][v] = fma(a[u], b[v], acc[u][v]);
          } else {
            const double d = a[u] - b[v];
            acc[u][v] = fma(d, d, acc[u][v]);
          }
        }
    }
    __syncthreads();
  }
  double mx = 0.0, sm = 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
      if (i < C && j < C) {
        const double dij = D[(long long)i * ldd + j];
        const double err = mode == 0 ? fabs(acc[u][v] - (1.0 - dij)) : fabs(sqrt(acc[u][v]) - dij);
        mx = fmax(mx, err);
        sm += err;
      }
    }
  rmax[tid] = mx;
  rsum[tid] = sm;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) { rmax[tid] = fmax(rmax[tid], rmax[tid + s]); rsum[tid] += rsum[tid + s]; }
    __syncthreads();
  }
  if (tid == 0) {
    const long long tile = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    ws[2 * tile] = rmax[0];
    ws[2 * tile + 1] = rsum[0];
  }
}

__global__ void __launch_bounds__(256) deviation_final_kernel(const double* __restrict__ ws, long long tiles, long long count,
                                                              double* __restrict__ out) {
  pdl_grid_sync();
  __shared__ double rmax[256], rsum[256];
  const int tid = threadIdx.x;
  double mx = 0.0, sm = 0.0;
  for (long long e = tid; e < tiles; e += 256) { mx = fmax(mx, ws[2 * e]); sm += ws[2 * e + 1]; }
  rmax[tid] = mx;
  rsum[tid] = sm;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) { rmax[tid] = fmax(rmax[tid], rmax[tid + s]); rsum[tid] += rsum[tid + s]; }
    __syncthreads();
  }
  if (tid == 0) { out[0] = rmax[0]; out[1] = rsum[0] / (double)count; }
}

inline int grid_for(long long total) { return (int)std::min<long long>(ceil_div<long long>(total, 256), 8LL * sm_count()); }

}  // namespace se

using namespace se;

extern "C" int se_lcs_height_table(const int32_t* offsets, const int32_t* ancestors, const int32_t* heights, int max_height,
                                   int C, int max_len, double* D, int64_t ldd, void* stream) {
  SE_REQUIRE(offsets && ancestors && heights && D, "null pointer");
  SE_REQUIRE(C > 0 && ldd >= C, "need C >= 1 and ldd >= C");
  SE_REQUIRE(max_height > 0, "need max_height >= 1");
  if (max_len > LCS_MAXLEN) {
    se::set_error("se_lcs_height_table: a class has %d ancestors, the table supports up to %d", max_len, LCS_MAXLEN);
    return SE_ERR_UNSUPPORTED;
  }
  const int tiles = ceil_div(C, LCS_TILE);
  launch(lcs_height_kernel, dim3(tiles, tiles), dim3(LCS_TILE, LCS_TILE), 0, as_stream(stream), (const int*)offsets,
         (const int*)ancestors, (const int*)heights, max_height, C, D, (long long)ldd);
  return check_launch("lcs_height_kernel");
}

extern "C" int se_cholesky_f64(double* A, int64_t lda, int n, int32_t* status, void* stream) {
  SE_REQUIRE(A && status, "null pointer");
  SE_REQUIRE(n > 0 && lda >= n, "need n >= 1 and lda >= n");
  cudaStream_t st = as_stream(stream);
  if (cudaMemsetAsync(status, 0xff, sizeof(int32_t), st) != cudaSuccess) return check_launch("se_cholesky_f64: status");
  for (int k0 = 0; k0 < n; k0 += CH_NB) {
    launch(chol_panel_kernel, dim3(1), dim3(256), 0, st, A, (long long)lda, n, k0, (int*)status);
    int rc = check_launch("chol_panel_kernel");
    if (rc) return rc;
    const int rest = n - k0 - CH_NB;
    if (rest <= 0) break;
    launch(chol_trsm_kernel, dim3(ceil_div(rest, CH_TRSM_ROWS)), dim3(CH_TRSM_ROWS), 0, st, A, (long long)lda, n, k0);
    if ((rc = check_launch("chol_trsm_kernel"))) return rc;
    const int tiles = ceil_div(rest, CH_TILE);
    launch(chol_update_kernel, dim3(tiles, tiles), dim3(128), 0, st, A, (long long)lda, n, k0);
    if ((rc = check_launch("chol_update_kernel"))) return rc;
  }
  launch(zero_upper_kernel, dim3(grid_for((long long)n * n)), dim3(256), 0, st, A, (long long)lda, n);
  return check_launch("zero_upper_kernel");
}

extern "C" int se_class_gram_f64(const double* D, int64_t ldd, int C, int op, double* out, int64_t ldo, void* stream) {
  SE_REQUIRE(D && out, "null pointer");
  SE_REQUIRE(op == SE_GRAM_SIM || op == SE_GRAM_SPHERES, "unknown op");
  SE_REQUIRE(C >= (op == SE_GRAM_SIM ? 1 : 2) && ldd >= C && ldo >= C - op, "bad sizes");
  const long long n = op == SE_GRAM_SIM ? C : C - 1;
  launch(class_gram_kernel, dim3(grid_for(n * n)), dim3(256), 0, as_stream(stream), D, (long long)ldd, C, op, out,
         (long long)ldo);
  return check_launch("class_gram_kernel");
}

extern "C" int se_column_op_f64(double* X, int64_t ldx, int m, int n, int op, double* out, void* stream) {
  SE_REQUIRE(X, "null pointer");
  SE_REQUIRE(op == SE_COL_SQNORM || op == SE_COL_CENTER, "unknown op");
  SE_REQUIRE(op != SE_COL_SQNORM || out, "SE_COL_SQNORM needs out");
  SE_REQUIRE(m > 0 && n > 0 && ldx >= n, "bad sizes");
  launch(column_op_kernel, dim3(ceil_div(n, 128)), dim3(128), 0, as_stream(stream), X, (long long)ldx, m, n, op, out);
  return check_launch("column_op_kernel");
}

extern "C" int se_gather_columns_f64(const double* X, int64_t ldx, int m, const int32_t* cols, int k, double* Y, int64_t ldy,
                                     void* stream) {
  SE_REQUIRE(X && cols && Y, "null pointer");
  SE_REQUIRE(m > 0 && k > 0 && ldy >= k, "bad sizes");
  launch(gather_columns_kernel, dim3(grid_for((long long)m * k)), dim3(256), 0, as_stream(stream), X, (long long)ldx, m,
         (const int*)cols, k, Y, (long long)ldy);
  return check_launch("gather_columns_kernel");
}

extern "C" int se_row_normalize_f64(double* X, int64_t ldx, int m, int n, void* stream) {
  SE_REQUIRE(X, "null pointer");
  SE_REQUIRE(m > 0 && n > 0 && ldx >= n, "bad sizes");
  launch(row_normalize_kernel, dim3(ceil_div(m, 8)), dim3(256), 0, as_stream(stream), X, (long long)ldx, m, n);
  return check_launch("row_normalize_kernel");
}

static int jacobi_blocks(int n) { const int b = ceil_div(n, JB); return b + (b & 1); }

extern "C" int64_t se_jacobi_columns_workspace_bytes(int m, int n) {
  (void)m;
  const long long pairs = jacobi_blocks(n) / 2;
  return (pairs * JP * JP * (long long)sizeof(double) + (pairs + 1) * (long long)sizeof(int) + 255) / 256 * 256;
}

extern "C" int se_jacobi_columns_f64(double* X, int64_t ldx, int m, int n, int max_sweeps, int32_t* sweeps, void* workspace,
                                     void* stream) {
  SE_REQUIRE(X && sweeps && workspace, "null pointer");
  SE_REQUIRE(m > 0 && n > 0 && ldx >= n && max_sweeps > 0, "bad sizes");
  cudaStream_t st = as_stream(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
    se::set_error("se_jacobi_columns_f64: the iteration synchronises with its stream and cannot be captured");
    return SE_ERR_ARG;
  }
  const int nbk = jacobi_blocks(n), pairs = nbk / 2;
  double* V = static_cast<double*>(workspace);
  int* rotated = reinterpret_cast<int*>(V + (long long)pairs * JP * JP);
  int* notconv = rotated + pairs;
  const double tol = (double)n * 2.220446049250313e-16;
  *sweeps = 0;
  for (int sweep = 1; sweep <= max_sweeps; ++sweep) {
    if (cudaMemsetAsync(notconv, 0, sizeof(int), st) != cudaSuccess) return check_launch("se_jacobi_columns_f64: flag");
    for (int round = 0; round < nbk - 1; ++round) {
      launch(jacobi_gram_kernel, dim3(pairs), dim3(JG_WARPS * 32), 0, st, (const double*)X, (long long)ldx, m, n, nbk, round,
             tol, V, rotated, notconv);
      int rc = check_launch("jacobi_gram_kernel");
      if (rc) return rc;
      launch(jacobi_apply_kernel, dim3(pairs, ceil_div(m, JA_ROWS)), dim3(128), 0, st, X, (long long)ldx, m, n, nbk, round,
             (const double*)V, (const int*)rotated);
      if ((rc = check_launch("jacobi_apply_kernel"))) return rc;
    }
    int host = 0;
    if (cudaMemcpyAsync(&host, notconv, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
      return check_launch("se_jacobi_columns_f64: flag");
    *sweeps = sweep;
    if (!host) return SE_OK;
  }
  se::set_error("se_jacobi_columns_f64: not converged after %d sweeps", max_sweeps);
  return SE_ERR_NOT_CONVERGED;
}

extern "C" int64_t se_embedding_deviation_workspace_bytes(int C) {
  const long long t = ceil_div(C, DV_T);
  return (2 * t * t * (long long)sizeof(double) + 255) / 256 * 256;
}

extern "C" int se_embedding_deviation_f64(const double* E, int64_t lde, int C, int dim, const double* D, int64_t ldd, int mode,
                                          double* out, void* workspace, void* stream) {
  SE_REQUIRE(E && D && out && workspace, "null pointer");
  SE_REQUIRE(mode == SE_DEV_SIM || mode == SE_DEV_DIST, "unknown mode");
  SE_REQUIRE(C > 0 && dim >= 0 && lde >= dim && ldd >= C, "bad sizes");
  cudaStream_t st = as_stream(stream);
  const int t = ceil_div(C, DV_T);
  double* ws = static_cast<double*>(workspace);
  launch(deviation_tile_kernel, dim3(t, t), dim3(256), 0, st, E, (long long)lde, C, dim, D, (long long)ldd, mode, ws);
  int rc = check_launch("deviation_tile_kernel");
  if (rc) return rc;
  launch(deviation_final_kernel, dim3(1), dim3(256), 0, st, (const double*)ws, (long long)t * t, (long long)C * C, out);
  return check_launch("deviation_final_kernel");
}
