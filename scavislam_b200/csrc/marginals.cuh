// marginals.cuh -- blocks of S^-1 from the block Cholesky factor of a BA handle's reduced system (marginals.cu), shared
// by svs_chol6_solve_blocks / _pattern (chol6.cu) and svs_ba_covariance (ba_host.cu)
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

#include "ba_types.cuh"

namespace svs {

// Device and pinned scratch of the inversion, grown on demand and kept by its owner across calls
struct InvScratch {
  double* zx = nullptr; size_t zx_cap = 0;                          // Z [nblk][36] | column solves [ncols][72 P]
  double* dinv = nullptr; size_t dinv_cap = 0;                      // D_j^-1 [P][36]
  char* d_req = nullptr; char* h_req = nullptr; size_t req_cap = 0;   // gather sources [n] | solved columns [ncols]
  int n = 0;                                                        // requests routed by the last invert()
  void release();
};

// Enqueues on `st`, behind a factor of d's reduced system that kept L_jj^-1 in d.Linv (launch_solve with keep_diag, or
// k_solve_general when general != 0): Z = S^-1 on the factor's pattern into w->zx, and the solves of the block columns
// that the n requests (req_r[k], req_c[k]) (poses) need outside that pattern.  tbl [P*P] and pos [P] are host copies
// of d.tbl and d.pos.  Nothing is waited for.  Kernels return at once when the factor failed (LmCtl::chol_fail).
cudaError_t invert(const BaDev& d, int general, const int* tbl, const int* pos, int n, const int* req_r, const int* req_c,
                   InvScratch* w, cudaStream_t st, int* in_pattern, int* ncols);
// The blocks the last invert() routed into out [n][36], each column-major (all zero when the factor failed)
cudaError_t gather(const BaDev& d, const InvScratch& w, double* out, cudaStream_t st);

}  // namespace svs
