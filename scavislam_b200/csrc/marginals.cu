// marginals.cu -- blocks of S^-1 from the block Cholesky factor of a BA handle's reduced system (marginals.cuh).
//
// The factor, written S = Lt D Lt^T with Lt_ij = N_ij = L_ij L_jj^-1 (unit lower) and D_j = L_jj L_jj^T, gives
// Z = S^-1 on the pattern of the factor by the Takahashi recurrences, over the columns in reverse elimination order
// (R_j = the sub-diagonal rows of column j):
//     Z_ij = - sum_{k in R_j} Z_ik N_kj   (i in R_j),      Z_jj = D_j^-1 - sum_{k in R_j} Z_kj^T N_kj.
// For i, k in R_j the block (i, k) lies in the factor's pattern, so every block the factor stores gets its inverse
// block (k_chol6_selinv).  A requested block outside the pattern comes from a solve S X = E_c of its column
// (k_chol6_inv_cols).  The recurrences read N from BaDev::Nrow (k_solve writes it for its backward pass; after
// k_solve_general, k_chol6_form_n forms it from S and Linv) and D_j^-1 = Linv_j^T Linv_j (k_solve's kDiag instance
// stores Linv as k_solve_general does).
#include <cstring>
#include <vector>

#include "handle.cuh"
#include "marginals.cuh"

namespace svs {

namespace {

// D_j^-1 = Linv_j^T Linv_j for every column (Linv_j = L_jj^-1, row-major lower triangular); exactly symmetric
__global__ void k_chol6_dinv(int P, const double* __restrict__ Linv, double* __restrict__ Dinv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 36 * P) return;
  const int j = i / 36, e = i - 36 * j, r = e / 6, c = e - 6 * r;
  const double* Li = Linv + 36 * (size_t)j;
  double s = 0.;
  for (int q = max(r, c); q < 6; ++q) s = fma(Li[6 * q + r], Li[6 * q + c], s);
  Dinv[i] = s;
}

// After k_solve_general (which leaves L_ij in S and L_jj^-1 in Linv): N_ij = L_ij L_jj^-1 into Nrow, laid out as
// k_solve's forward pass writes it (the transposed block at the block's row-major position)
__global__ void k_chol6_form_n(int nblk, const int* __restrict__ rowpos, const int* __restrict__ rcol,
                               const double* __restrict__ S, const double* __restrict__ Linv, double* __restrict__ Nrow) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 36ll * nblk) return;
  const int b = (int)(i / 36), e = (int)(i - 36ll * b), r = e / 6, c = e - 6 * r;
  const int p = rowpos[b];
  if (p < 0) return;   // a diagonal block
  const double* L = S + 36 * (size_t)b + 6 * r;
  const double* Li = Linv + 36 * (size_t)rcol[p];
  double s = 0.;
  for (int q = c; q < 6; ++q) s = fma(L[q], Li[6 * q + c], s);
  Nrow[36 * (size_t)p + 6 * c + r] = s;
}

// The Takahashi recurrences (header comment) over the columns [j0, j1) in reverse, into Z in S's block layout.
// sep = 1: one CTA takes the separator columns [branch_ptr[G], P); sep = 0: CTA g takes branch g, which depends
// only on itself and the separator (launched after the separator).  Inside a column the 36 |R_j| elements of
// the Z_ij are spread over the threads, each a sum over the |R_j| products Z_ik N_kj; Z_ik is found through
// perm and tbl (transposed when the table says the stored block is (k, i)).
constexpr int kSelThreads = 256;
__global__ void __launch_bounds__(kSelThreads) k_chol6_selinv(BaDev d, const double* __restrict__ Dinv, double* Z, int sep) {
  if (d.ctl->chol_fail) return;
  const int P = d.P, G = d.nbranch, t = threadIdx.x;
  const int j0 = sep ? d.branch_ptr[G] : d.branch_ptr[blockIdx.x];
  const int j1 = sep ? P : d.branch_ptr[blockIdx.x + 1];
  for (int j = j1 - 1; j >= j0; --j) {
    const int base = d.col_ptr[j] + 1, nb = d.col_ptr[j + 1] - base;
    for (int o = t; o < 36 * nb; o += kSelThreads) {
      const int a = o / 36, e = o - 36 * a, r = e / 6, c = e - 6 * r;
      const size_t row_a = (size_t)__ldg(d.perm + __ldg(d.row_idx + base + a)) * P;
      double s = 0.;
      for (int k = 0; k < nb; ++k) {
        const int tk = __ldg(d.tbl + row_a + __ldg(d.perm + __ldg(d.row_idx + base + k)));
        const double* Zak = Z + 36 * (size_t)(tk >> 1) + ((tk & 1) ? r : 6 * r);   // row r of Z_ak
        const int zq = (tk & 1) ? 6 : 1;
        const double* Nk = d.Nrow + 36 * (size_t)__ldg(d.rowpos + base + k) + 6 * c;   // column c of N_kj
#pragma unroll
        for (int q = 0; q < 6; ++q) s = fma(Zak[q * zq], __ldg(Nk + q), s);
      }
      Z[36 * (size_t)(base + a) + e] = -s;
    }
    __syncthreads();
    if (t < 36) {   // Z_jj: the lower triangle, mirrored
      const int r = t / 6, c = t - 6 * r;
      if (r >= c) {
        double s = Dinv[36 * (size_t)j + t];
        for (int a = 0; a < nb; ++a) {
          const double* Za = Z + 36 * (size_t)(base + a) + r;   // column r of Z_aj
          const double* Na = d.Nrow + 36 * (size_t)__ldg(d.rowpos + base + a) + 6 * c;
#pragma unroll
          for (int q = 0; q < 6; ++q) s = fma(-Za[6 * q], __ldg(Na + q), s);
        }
        Z[36 * (size_t)(base - 1) + t] = s;
        Z[36 * (size_t)(base - 1) + 6 * c + r] = s;
      }
    }
    __syncthreads();
  }
}

// Columns of S^-1 outside the factor's pattern: CTA s solves S X = E_c for pose c = cols[s] (six right-hand sides)
// with the same factor -- forward through N (row-major, from the column's position on: Y is zero before it), D^-1,
// backward through N^T -- into X + 72 P s: [P][36] X (row-major 6x6 per position), then [P][36] D^-1 Y.
// Thread t < 36 owns element (t / 6, t % 6) of the current position's block.
constexpr int kColThreads = 64;
__global__ void __launch_bounds__(kColThreads) k_chol6_inv_cols(BaDev d, const double* __restrict__ Dinv,
                                                                const int* __restrict__ cols, double* X) {
  if (d.ctl->chol_fail) return;
  const int P = d.P, t = threadIdx.x, jc = d.pos[cols[blockIdx.x]];
  double* Y = X + 72 * (size_t)P * blockIdx.x;
  double* W = Y + 36 * (size_t)P;
  const bool on = t < 36;
  const int r = t / 6, e = t - 6 * r;
  for (int i = t; i < 36 * jc; i += kColThreads) { Y[i] = 0.; W[i] = 0.; }
  for (int j = jc; j < P; ++j) {   // Y_j = E_j - sum_k N_jk Y_k
    if (on) {
      double s = (j == jc && r == e) ? 1. : 0.;
      for (int p = __ldg(d.rptr + j); p < __ldg(d.rptr + j + 1); ++p) {
        const int k = __ldg(d.rcol + p);
        if (k < jc) break;   // columns descend inside a row
        const double* N = d.Nrow + 36 * (size_t)p + r;   // row r of N_jk
        const double* Yk = Y + 36 * (size_t)k + e;
#pragma unroll
        for (int q = 0; q < 6; ++q) s = fma(-__ldg(N + 6 * q), Yk[6 * q], s);
      }
      Y[36 * (size_t)j + t] = s;
    }
    __syncthreads();
    if (on) {
      double w = 0.;
#pragma unroll
      for (int q = 0; q < 6; ++q) w = fma(Dinv[36 * (size_t)j + 6 * r + q], Y[36 * (size_t)j + 6 * q + e], w);
      W[36 * (size_t)j + t] = w;
    }
  }
  __syncthreads();
  for (int j = P - 1; j >= 0; --j) {   // X_j = W_j - sum_{i in R_j} N_ij^T X_i, over Y
    if (on) {
      double s = W[36 * (size_t)j + t];
      for (int b = __ldg(d.col_ptr + j) + 1; b < __ldg(d.col_ptr + j + 1); ++b) {
        const double* N = d.Nrow + 36 * (size_t)__ldg(d.rowpos + b) + 6 * r;   // column r of N_ij
        const double* Xi = Y + 36 * (size_t)__ldg(d.row_idx + b) + e;
#pragma unroll
        for (int q = 0; q < 6; ++q) s = fma(-__ldg(N + q), Xi[6 * q], s);
      }
      Y[36 * (size_t)j + t] = s;
    }
    __syncthreads();
  }
}

// Requested block k into out[k] column-major: src[k] = (offset of the row-major 6x6 in ZX) << 1 | transpose.
// All zero when the factor failed.
__global__ void k_chol6_gather(int n, const long long* __restrict__ src, const double* __restrict__ ZX,
                               const int* __restrict__ fail, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 36ll * n) return;
  const int k = (int)(i / 36), e = (int)(i - 36ll * k), c = e / 6, r = e - 6 * c;   // element (r, c) of block k
  const long long s = src[k];
  const double* B = ZX + (s >> 1);
  out[i] = *fail ? 0. : ((s & 1) ? B[6 * c + r] : B[6 * r + c]);
}

}  // namespace

void InvScratch::release() {
  for (double* p : {zx, dinv})
    if (p) cudaFree(p);
  if (d_req) cudaFree(d_req);
  if (h_req) cudaFreeHost(h_req);
  *this = InvScratch{};
}

cudaError_t invert(const BaDev& d, int general, const int* tbl, const int* pos, int n, const int* req_r, const int* req_c,
                   InvScratch* w, cudaStream_t st, int* in_pattern, int* ncols_out) {
  const int P = d.P, nblk = d.nblk;
  // where each request is served from: Z when the block lies in the factor's pattern, else the solve of its column
  // (or, transposed, of its row when that column is solved anyway)
  std::vector<long long> src(n);
  std::vector<int> cols, slot(P, -1);
  int inp = 0;
  for (int k = 0; k < n; ++k) {
    const int r = req_r[k], c = req_c[k], t = tbl[(size_t)r * P + c];
    if (t >= 0) {
      src[k] = (36ll * (t >> 1)) << 1 | (t & 1);
      ++inp;
      continue;
    }
    if (slot[c] < 0 && slot[r] >= 0) {
      src[k] = (36ll * nblk + 72ll * P * slot[r] + 36ll * pos[c]) << 1 | 1;
      continue;
    }
    if (slot[c] < 0) { slot[c] = (int)cols.size(); cols.push_back(c); }
    src[k] = (36ll * nblk + 72ll * P * slot[c] + 36ll * pos[r]) << 1;
  }
  const int ncols = (int)cols.size();
  *in_pattern = inp;
  *ncols_out = ncols;
  w->n = n;
  cudaError_t e;
  if ((e = grow(36 * (size_t)nblk + 72 * (size_t)P * ncols, &w->zx_cap, &w->zx)) != cudaSuccess) return e;
  if ((e = grow(36 * (size_t)P, &w->dinv_cap, &w->dinv)) != cudaSuccess) return e;
  const size_t src_bytes = (size_t)n * sizeof(long long), req_bytes = src_bytes + (size_t)ncols * sizeof(int);
  if ((e = grow(req_bytes, &w->req_cap, &w->d_req, &w->h_req)) != cudaSuccess) return e;
  memcpy(w->h_req, src.data(), src_bytes);
  memcpy(w->h_req + src_bytes, cols.data(), (size_t)ncols * sizeof(int));
  if ((e = cudaMemcpyAsync(w->d_req, w->h_req, req_bytes, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if (general)
    k_chol6_form_n<<<(unsigned)((36ll * nblk + 255) / 256), 256, 0, st>>>(nblk, d.rowpos, d.rcol, d.S, d.Linv, d.Nrow);
  k_chol6_dinv<<<(36 * P + 255) / 256, 256, 0, st>>>(P, d.Linv, w->dinv);
  const int G = d.nbranch;
  if (G > 1) k_chol6_selinv<<<1, kSelThreads, 0, st>>>(d, w->dinv, w->zx, 1);   // the separator first
  k_chol6_selinv<<<G, kSelThreads, 0, st>>>(d, w->dinv, w->zx, 0);
  if (ncols > 0)
    k_chol6_inv_cols<<<ncols, kColThreads, 0, st>>>(d, w->dinv, reinterpret_cast<const int*>(w->d_req + src_bytes),
                                                    w->zx + 36 * (size_t)nblk);
  return cudaGetLastError();
}

cudaError_t gather(const BaDev& d, const InvScratch& w, double* out, cudaStream_t st) {
  const size_t nout = 36 * (size_t)w.n;
  if (nout == 0) return cudaSuccess;
  k_chol6_gather<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>(w.n, reinterpret_cast<const long long*>(w.d_req), w.zx,
                                                                   &d.ctl->chol_fail, out);
  return cudaGetLastError();
}

}  // namespace svs
