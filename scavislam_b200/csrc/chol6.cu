// chol6.cu -- svs_chol6: the device block Cholesky of the BA path for a caller's own 6x6-block system
// (include/svs_b200.h).  It stands where g2o::LinearSolverCSparse<Matrix6d> stands in the reference
// (slam_graph.cpp:55-60): LinearSolver::solve(A, x, b) on the upper triangle of A in block CCS.
//
// The handle owns an internal svs_ba.  A new block pattern becomes that handle's problem: P identity poses, no
// landmarks, no edges, the pattern's off-diagonal pairs prescribed with svs_ba_set_structure.  Its set_problem does
// the symbolic analysis (minimum-degree order, two-ended split, solver choice) and keeps it cached by the P x P
// pattern.  Every solve then clears S, scatters the caller's blocks and right-hand side into it (k_chol6_scatter)
// and runs the BA handle's solve with lambda = 0.
//
// Marginals (LinearSolver::solveBlocks / solvePattern, as LinearSolverCSparse computes them with
// MarginalCovarianceCholesky): the same factor with L_jj^-1 kept, inverted on its pattern by the selected inversion
// of marginals.cu, which svs_ba_covariance shares.
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/svs_b200.h"
#include "ba_types.cuh"
#include "handle.cuh"
#include "internal.cuh"
#include "marginals.cuh"

using namespace svs;

namespace {

// The caller's upper blocks (column-major 6x6, block k couples poses rc[k].x <= rc[k].y) into S (lower blocks in
// elimination order, row-major, rows <-> the pose the table names) through the analysis' (row pose, col pose) ->
// block << 1 | transpose table.  A diagonal block is read from its upper triangle and written whole.  The threads
// past the blocks load the right-hand side: bp = b, bc = 0 (the solve factors bp - bc).
__global__ void k_chol6_scatter(int P, int nnzb, const int2* __restrict__ rc, const double* __restrict__ blocks,
                                const double* __restrict__ b, const int* __restrict__ tbl, double* __restrict__ S,
                                double* __restrict__ bp, double* __restrict__ bc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nS = 36ll * nnzb;
  if (i < nS) {
    const int k = (int)(i / 36), e = (int)(i - 36ll * k), c = e / 6, r = e - 6 * c;   // element (r, c) of block k
    const int2 q = rc[k];
    const int t = tbl[(size_t)q.x * P + q.y];
    double* dst = S + 36 * (size_t)(t >> 1);
    const double v = blocks[i];
    if (q.x == q.y) {
      if (r <= c) { dst[6 * r + c] = v; dst[6 * c + r] = v; }
    } else {
      dst[(t & 1) ? 6 * c + r : 6 * r + c] = v;
    }
  } else if (i < nS + 6ll * P) {
    const int j = (int)(i - nS);
    bp[j] = b[j];
    bc[j] = 0.;
  }
}

}  // namespace

struct svs_chol6 : svs::Handle {
  svs_ba* ba = nullptr;
  // pattern of the problem on the internal BA handle (P < 0: none)
  int P = -1;
  std::vector<int> col_ptr, row_idx;
  int2* d_rc = nullptr; size_t rc_cap = 0;                       // (row, col) pose of every upper block
  double* d_in = nullptr; double* h_in = nullptr; size_t in_cap = 0;   // host inputs: blocks | b
  double* h_x = nullptr; size_t x_cap = 0;                      // pinned read-out of x
  int* h_fail = nullptr;                                         // pinned LmCtl::chol_fail
  cudaEvent_t ev[2] = {};
  // marginals
  std::vector<int> tbl, pos;                                     // host copies of the analysis' table and positions
  InvScratch inv;
  double* d_out = nullptr; double* h_out = nullptr; size_t out_cap = 0;   // requested blocks of a host-memory call
};

namespace {

// The checks of the header comment, before anything is enqueued.  `ptrs` are the entry point's array arguments
// besides the pattern (named `what` in the messages): never null, and on the handle's device when on_device != 0.
int validate(svs_chol6* h, const char* fn, int P, const int* col_ptr, const int* row_idx,
             std::initializer_list<const void*> ptrs, const char* what, int on_device) {
  const std::string f = std::string(fn) + ": ";
  if (P < 0) return fail(h, SVS_ERR_INVALID, f + "P < 0");
  if (!col_ptr) return fail(h, SVS_ERR_INVALID, f + "null col_ptr");
  if (col_ptr[0] != 0) return fail(h, SVS_ERR_INVALID, f + "col_ptr[0] != 0");
  for (int j = 0; j < P; ++j)
    if (col_ptr[j + 1] < col_ptr[j]) return fail(h, SVS_ERR_INVALID, f + "col_ptr decreases at column " + std::to_string(j));
  if (P == 0) return SVS_OK;
  bool null = !row_idx;
  for (const void* p : ptrs) null = null || !p;
  if (null) return fail(h, SVS_ERR_INVALID, f + "null row_idx, " + what);
  for (int j = 0; j < P; ++j) {
    const int b0 = col_ptr[j], b1 = col_ptr[j + 1];
    for (int k = b0; k < b1; ++k) {
      const int r = row_idx[k];
      if (r < 0 || r > j)
        return fail(h, SVS_ERR_INVALID, f + "row " + std::to_string(r) + " in column " + std::to_string(j) +
                                             " is not in the upper triangle");
      if (k > b0 && r <= row_idx[k - 1])
        return fail(h, SVS_ERR_INVALID, f + "rows of column " + std::to_string(j) + " are not strictly ascending");
    }
    if (b1 == b0 || row_idx[b1 - 1] != j)
      return fail(h, SVS_ERR_INVALID, f + "column " + std::to_string(j) + " has no diagonal block");
  }
  if (on_device) {
    for (const void* p : ptrs)
      if (!svs::on_device(h->device, p))
        return fail(h, SVS_ERR_INVALID, f + "on_device = 1 but " + what + " is not memory of the handle's device");
  }
  return SVS_OK;
}

// Makes the caller's pattern the internal BA handle's problem (the handle decides whether to re-analyse).
int set_pattern(svs_chol6* h, const char* fn, int P, const int* col_ptr, const int* row_idx) {
  h->P = -1;
  const int nnzb = col_ptr[P];
  std::vector<int> pi, pj;
  std::vector<int2> rc(nnzb);
  for (int j = 0; j < P; ++j)
    for (int k = col_ptr[j]; k < col_ptr[j + 1]; ++k) {
      rc[k] = make_int2(row_idx[k], j);
      if (row_idx[k] != j) { pi.push_back(row_idx[k]); pj.push_back(j); }
    }
  int rc_ = svs_ba_set_structure(h->ba, (int)pi.size(), pi.data(), pj.data());
  if (rc_ == SVS_OK) {
    std::vector<double> T((size_t)7 * P, 0.);
    for (int p = 0; p < P; ++p) T[7 * (size_t)p + 3] = 1.;   // identity: q = (0, 0, 0, 1), t = 0
    const svs_cam cam{1., 0., 0., 1.};
    rc_ = svs_ba_set_problem(h->ba, P, T.data(), nullptr, 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                             nullptr, nullptr, nullptr, nullptr, &cam);
  }
  if (rc_ != SVS_OK) return fail(h, rc_, std::string(fn) + ": " + svs_last_error(h->ba));
  SVS_CK(h, grow((size_t)nnzb, &h->rc_cap, &h->d_rc));
  const BaDev* d = nullptr; cudaStream_t st = nullptr; int hits = 0;
  if ((rc_ = ba_system_on_device(h->ba, &d, &st, &hits))) return fail(h, rc_, std::string(fn) + ": no problem on the internal handle");
  SVS_CK(h, cudaMemcpyAsync(h->d_rc, rc.data(), (size_t)nnzb * sizeof(int2), cudaMemcpyHostToDevice, st));
  h->tbl.resize((size_t)P * P);
  h->pos.resize(P);
  SVS_CK(h, cudaMemcpyAsync(h->tbl.data(), d->tbl, h->tbl.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  SVS_CK(h, cudaMemcpyAsync(h->pos.data(), d->pos, (size_t)P * sizeof(int), cudaMemcpyDeviceToHost, st));
  SVS_CK(h, cudaStreamSynchronize(st));   // rc is a pageable temporary
  h->P = P;
  h->col_ptr.assign(col_ptr, col_ptr + P + 1);
  h->row_idx.assign(row_idx, row_idx + nnzb);
  return SVS_OK;
}

// What factor() enqueued: the internal handle's system, its stream, which solver ran, whether the analysis was reused.
struct Factor {
  const BaDev* d = nullptr;
  cudaStream_t st = nullptr;
  int general = 0, reused = 1;
};

// The part the entry points share, after validate(): make the pattern the internal handle's problem (re-analysing
// only when it changed), stage the inputs, clear S, scatter, and enqueue the factor and solve with lambda = 0.
// b == nullptr: a zero right-hand side.  keep_diag: leave L_jj^-1 in Linv (k_solve's kDiag instance).  ev[0] is
// recorded before the scatter; nothing is waited for.
int factor(svs_chol6* h, const char* fn, int P, const int* col_ptr, const int* row_idx, const double* blocks,
           const double* b, int on_device, int keep_diag, Factor* f) {
  cudaSetDevice(h->device);
  const int nnzb = col_ptr[P];
  if (!(P == h->P && memcmp(col_ptr, h->col_ptr.data(), sizeof(int) * (P + 1)) == 0 &&
        memcmp(row_idx, h->row_idx.data(), sizeof(int) * (size_t)nnzb) == 0)) {
    const BaDev* d0 = nullptr; cudaStream_t s0 = nullptr; int hits0 = -1;
    if (ba_system_on_device(h->ba, &d0, &s0, &hits0) != SVS_OK) hits0 = -1;
    if (int rc = set_pattern(h, fn, P, col_ptr, row_idx)) return rc;
    const BaDev* d1 = nullptr; cudaStream_t s1 = nullptr; int hits1 = 0;
    ba_system_on_device(h->ba, &d1, &s1, &hits1);
    f->reused = hits0 >= 0 && hits1 > hits0;
  }
  const BaDev* d = nullptr; cudaStream_t st = nullptr; int hits = 0;
  if (int rc = ba_system_on_device(h->ba, &d, &st, &hits)) return fail(h, rc, std::string(fn) + ": no problem on the internal handle");
  f->d = d;
  f->st = st;
  const size_t nA = 36 * (size_t)nnzb, n = 6 * (size_t)P;
  const double* d_blocks = blocks;
  const double* d_b = b;
  if (!on_device) {   // staged in pinned memory, one copy
    SVS_CK(h, grow(nA + n, &h->in_cap, &h->d_in, &h->h_in));
    memcpy(h->h_in, blocks, nA * sizeof(double));
    if (b) memcpy(h->h_in + nA, b, n * sizeof(double));
    else memset(h->h_in + nA, 0, n * sizeof(double));
    SVS_CK(h, cudaMemcpyAsync(h->d_in, h->h_in, (nA + n) * sizeof(double), cudaMemcpyHostToDevice, st));
    d_blocks = h->d_in;
    d_b = h->d_in + nA;
  } else if (!b) {
    SVS_CK(h, grow(n, &h->in_cap, &h->d_in, &h->h_in));
    SVS_CK(h, cudaMemsetAsync(h->d_in, 0, n * sizeof(double), st));
    d_b = h->d_in;
  }
  SVS_CK(h, cudaEventRecord(h->ev[0], st));
  SVS_CK(h, cudaMemsetAsync(d->S, 0, 36 * (size_t)d->nblk * sizeof(double), st));   // the fill-in blocks start from zero
  const long long work = (long long)nA + (long long)n;
  k_chol6_scatter<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(P, nnzb, h->d_rc, d_blocks, d_b, d->tbl, d->S, d->bp, d->bc);
  SVS_CK(h, cudaGetLastError());
  if (int rc = ba_solve_system(h->ba, &f->general, keep_diag)) return fail(h, rc, std::string(fn) + ": " + svs_last_error(h->ba));
  return SVS_OK;
}

// The marginal entry points after validation: factor, invert on the factor's pattern, solve the columns the requests
// need outside it, gather the n blocks (req_r[k], req_c[k]) into out[k] (column-major), wait.
int invert(svs_chol6* h, const char* fn, int P, const int* col_ptr, const int* row_idx, const double* blocks, int n,
           const int* req_r, const int* req_c, double* out, int on_device, svs_chol6_inv_stats* stats) {
  Factor f;
  if (int rc = factor(h, fn, P, col_ptr, row_idx, blocks, nullptr, on_device, 1, &f)) return rc;
  const BaDev* d = f.d;
  const cudaStream_t st = f.st;
  int in_pattern = 0, ncols = 0;
  SVS_CK(h, svs::invert(*d, f.general, h->tbl.data(), h->pos.data(), n, req_r, req_c, &h->inv, st, &in_pattern, &ncols));
  SVS_CK(h, cudaEventRecord(h->ev[1], st));
  double* d_out = out;
  const size_t nout = 36 * (size_t)n;
  if (!on_device) {
    SVS_CK(h, grow(nout, &h->out_cap, &h->d_out, &h->h_out));
    d_out = h->d_out;
  }
  SVS_CK(h, gather(*d, h->inv, d_out, st));
  SVS_CK(h, cudaMemcpyAsync(h->h_fail, &d->ctl->chol_fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (!on_device) SVS_CK(h, cudaMemcpyAsync(h->h_out, d_out, nout * sizeof(double), cudaMemcpyDeviceToHost, st));
  SVS_CK(h, cudaStreamSynchronize(st));
  if (!on_device) memcpy(out, h->h_out, nout * sizeof(double));
  if (stats) {
    stats->P = P; stats->nnzb_A = col_ptr[P]; stats->nnzb_L = d->nblk; stats->nbranch = d->nbranch;
    stats->general = f.general; stats->symbolic_reused = f.reused;
    stats->n_in_pattern = in_pattern; stats->n_cols_solved = ncols;
    cudaEventElapsedTime(&stats->ms, h->ev[0], h->ev[1]);
  }
  return *h->h_fail ? 1 : 0;
}

}  // namespace

extern "C" {

int svs_chol6_create(int device, svs_chol6** out) {
  if (!out) return SVS_ERR_INVALID;
  *out = nullptr;
  svs_chol6* h = new svs_chol6();
  int rc = open_handle(h, device, false);
  const svs_ba_opts o{device, 0, {0, 0, 0, 0, 0, 0}};
  if (rc == SVS_OK) rc = svs_ba_create(&o, &h->ba);
  if (rc != SVS_OK) {
    delete h;
    return rc;
  }
  if (cudaMallocHost(&h->h_fail, sizeof(int)) != cudaSuccess ||
      cudaEventCreate(&h->ev[0]) != cudaSuccess || cudaEventCreate(&h->ev[1]) != cudaSuccess) {
    svs_chol6_destroy(h);
    return SVS_ERR_CUDA;
  }
  *out = h;
  return SVS_OK;
}

void svs_chol6_destroy(svs_chol6* h) {
  if (!h) return;
  begin_close(h);
  if (h->ba) svs_ba_destroy(h->ba);   // waits for the stream
  if (h->d_rc) cudaFree(h->d_rc);
  if (h->d_in) cudaFree(h->d_in);
  if (h->h_in) cudaFreeHost(h->h_in);
  if (h->h_x) cudaFreeHost(h->h_x);
  if (h->h_fail) cudaFreeHost(h->h_fail);
  h->inv.release();
  if (h->d_out) cudaFree(h->d_out);
  if (h->h_out) cudaFreeHost(h->h_out);
  for (auto& e : h->ev)
    if (e) cudaEventDestroy(e);
  delete h;
}

const char* svs_chol6_last_error(const svs_chol6* h) { return last_error(h); }

int svs_chol6_init(svs_chol6* h) {
  if (!h) return SVS_ERR_INVALID;
  h->P = -1;
  h->col_ptr.clear();
  h->row_idx.clear();
  ba_forget_symbolic(h->ba);
  return SVS_OK;
}

int svs_chol6_solve(svs_chol6* h, int P, const int* col_ptr, const int* row_idx, const double* blocks, const double* b,
                    double* x, int on_device, svs_chol6_stats* stats) {
  if (!h) return SVS_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  const char* fn = "svs_chol6_solve";
  if (int rc = validate(h, fn, P, col_ptr, row_idx, {blocks, b, x}, "blocks, b or x", on_device)) return rc;
  if (P == 0) return 0;
  Factor f;
  if (int rc = factor(h, fn, P, col_ptr, row_idx, blocks, b, on_device, 0, &f)) return rc;
  const size_t n = 6 * (size_t)P;
  SVS_CK(h, cudaEventRecord(h->ev[1], f.st));
  SVS_CK(h, cudaMemcpyAsync(h->h_fail, &f.d->ctl->chol_fail, sizeof(int), cudaMemcpyDeviceToHost, f.st));
  if (on_device) {
    SVS_CK(h, cudaMemcpyAsync(x, f.d->x, n * sizeof(double), cudaMemcpyDeviceToDevice, f.st));
  } else {
    SVS_CK(h, grow(n, &h->x_cap, (double**)nullptr, &h->h_x));
    SVS_CK(h, cudaMemcpyAsync(h->h_x, f.d->x, n * sizeof(double), cudaMemcpyDeviceToHost, f.st));
  }
  SVS_CK(h, cudaStreamSynchronize(f.st));
  if (!on_device) memcpy(x, h->h_x, n * sizeof(double));
  if (stats) {
    stats->P = P; stats->nnzb_A = col_ptr[P]; stats->nnzb_L = f.d->nblk; stats->nbranch = f.d->nbranch;
    stats->general = f.general; stats->symbolic_reused = f.reused;
    cudaEventElapsedTime(&stats->ms, h->ev[0], h->ev[1]);
  }
  return *h->h_fail ? 1 : 0;
}

int svs_chol6_solve_blocks(svs_chol6* h, int P, const int* col_ptr, const int* row_idx, const double* blocks,
                           double* inv_diag, int on_device, svs_chol6_inv_stats* stats) {
  if (!h) return SVS_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  const char* fn = "svs_chol6_solve_blocks";
  if (int rc = validate(h, fn, P, col_ptr, row_idx, {blocks, inv_diag}, "blocks or inv_diag", on_device)) return rc;
  if (P == 0) return 0;
  std::vector<int> diag(P);
  for (int p = 0; p < P; ++p) diag[p] = p;
  return invert(h, fn, P, col_ptr, row_idx, blocks, P, diag.data(), diag.data(), inv_diag, on_device, stats);
}

int svs_chol6_solve_pattern(svs_chol6* h, int P, const int* col_ptr, const int* row_idx, const double* blocks, int n,
                            const int* req_r, const int* req_c, double* out, int on_device, svs_chol6_inv_stats* stats) {
  if (!h) return SVS_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  const char* fn = "svs_chol6_solve_pattern";
  if (n < 0) return fail(h, SVS_ERR_INVALID, std::string(fn) + ": n < 0");
  if (n > 0 && (!req_r || !req_c || !out)) return fail(h, SVS_ERR_INVALID, std::string(fn) + ": null req_r, req_c or out");
  for (int k = 0; k < n; ++k)
    if (req_r[k] < 0 || req_r[k] >= P || req_c[k] < 0 || req_c[k] >= P)
      return fail(h, SVS_ERR_INVALID, std::string(fn) + ": request " + std::to_string(k) + " (" + std::to_string(req_r[k]) +
                                           ", " + std::to_string(req_c[k]) + ") is outside [0, P)");
  if (n == 0) return validate(h, fn, P, col_ptr, row_idx, {blocks}, "blocks", on_device);
  if (int rc = validate(h, fn, P, col_ptr, row_idx, {blocks, out}, "blocks or out", on_device)) return rc;
  return invert(h, fn, P, col_ptr, row_idx, blocks, n, req_r, req_c, out, on_device, stats);
}

}  // extern "C"
