// The g2o linear-solver adapter of INTEGRATION.md §1 with its marginal overrides (solveBlocks, solvePattern) against a
// minimal stand-in for the parts of g2o they touch (Matrix6d, MatrixXd, SparseBlockMatrix, LinearSolver).  Reads a
// system written by tests/test_chol6_marginals_gpu.py:
//   int32 P, int32 nnzb, int32 col_ptr[P + 1], int32 row_idx[nnzb], float64 blocks[nnzb][36] (column-major),
//   int32 n, int32 r[n], int32 c[n]
// builds a SparseBlockMatrix holding every block of A, and writes the P diagonal blocks of A^-1 from solveBlocks, then
// the n blocks (r[k], c[k]) from solvePattern, each column-major.  Exit 0 on success, 1 if not positive definite, 2 on
// bad input, 3 without a GPU.
#include <algorithm>
#include <cstdio>
#include <map>
#include <memory>
#include <stdexcept>
#include <utility>
#include <vector>

#include "svs_b200.hpp"

namespace g2o {
struct Matrix6d {   // Eigen::Matrix<double, 6, 6>: column-major storage
  enum { RowsAtCompileTime = 6, ColsAtCompileTime = 6 };
  double v[36] = {};
  double* data() { return v; }
  const double* data() const { return v; }
};
struct MatrixXd {   // Eigen::MatrixXd as SparseBlockMatrix<MatrixXd>::block(r, c, true) allocates it for pose blocks
  double v[36] = {};
  double* data() { return v; }
  const double* data() const { return v; }
};

template <typename MatrixType>
class SparseBlockMatrix {   // per block column: row block -> block, ordered by row
 public:
  typedef std::map<int, MatrixType*> IntBlockMap;
  explicit SparseBlockMatrix(int nblocks) : cols_(nblocks) {}
  ~SparseBlockMatrix() {
    for (auto& c : cols_)
      for (auto& rb : c) delete rb.second;
  }
  MatrixType* block(int r, int c, bool alloc) {
    auto it = cols_[c].find(r);
    if (it != cols_[c].end()) return it->second;
    return alloc ? (cols_[c][r] = new MatrixType()) : nullptr;
  }
  const std::vector<IntBlockMap>& blockCols() const { return cols_; }

 private:
  std::vector<IntBlockMap> cols_;
};

template <typename MatrixType>
class LinearSolver {
 public:
  virtual ~LinearSolver() {}
  virtual bool init() = 0;
  virtual bool solve(const SparseBlockMatrix<MatrixType>& A, double* x, double* b) = 0;
  virtual bool solveBlocks(double**& blocks, const SparseBlockMatrix<MatrixType>& A) { (void)blocks; (void)A; return false; }
  virtual bool solvePattern(SparseBlockMatrix<MatrixXd>& spinv, const std::vector<std::pair<int, int>>& blockIndices,
                            const SparseBlockMatrix<MatrixType>& A) {
    (void)spinv; (void)blockIndices; (void)A;
    return false;
  }
};
}  // namespace g2o

// The adapter of tests/cpp/chol6_main.cpp with the overrides of INTEGRATION.md inserted after solve()
template <typename MatrixType>
class LinearSolverSvs : public g2o::LinearSolver<MatrixType> {
  static_assert(MatrixType::RowsAtCompileTime == 6 && MatrixType::ColsAtCompileTime == 6, "6x6 pose blocks only");

 public:
  // LinearSolverCSparse::init() drops its symbolic factorisation because it cannot tell whether the next matrix
  // keeps the pattern.  svs_chol6 compares the pattern on every solve, so the analysis may outlive one optimize().
  // (Call solver_.init() here to re-analyse on every optimize() as CSparse does.)
  bool init() override { return true; }

  // A is the Schur complement g2o's BlockSolver built; only its upper triangle is handed over (fillCCS(..., true))
  bool solve(const g2o::SparseBlockMatrix<MatrixType>& A, double* x, double* b) override {
    const int P = (int)A.blockCols().size();
    col_ptr_.assign(1, 0);
    row_idx_.clear();
    blocks_.clear();
    for (int j = 0; j < P; ++j) {
      for (const auto& rb : A.blockCols()[j]) {   // ascending row blocks
        if (rb.first > j) break;
        row_idx_.push_back(rb.first);
        blocks_.insert(blocks_.end(), rb.second->data(), rb.second->data() + 36);
      }
      col_ptr_.push_back((int)row_idx_.size());
    }
    return solver_.solve(P, col_ptr_.data(), row_idx_.data(), blocks_.data(), x, b);   // false: not positive definite
  }
// ---- INTEGRATION.md overrides begin
  // The diagonal blocks of A^-1.  A null `blocks` is allocated here, one 6x6 array per block column, and belongs to
  // the caller afterwards.
  bool solveBlocks(double**& blocks, const g2o::SparseBlockMatrix<MatrixType>& A) override {
    const int P = upper(A);
    if (!blocks) {
      blocks = new double*[P];
      for (int i = 0; i < P; ++i) blocks[i] = new double[36];
    }
    inv_.resize(36 * (size_t)P);
    if (!solver_.solveBlocks(P, col_ptr_.data(), row_idx_.data(), blocks_.data(), inv_.data())) return false;
    for (int i = 0; i < P; ++i) std::copy(inv_.begin() + 36 * i, inv_.begin() + 36 * (i + 1), blocks[i]);
    return true;
  }

  // SparseOptimizer::computeMarginals -> BlockSolver::computeMarginals: the blocks (r, c) of A^-1 into spinv
  bool solvePattern(g2o::SparseBlockMatrix<g2o::MatrixXd>& spinv, const std::vector<std::pair<int, int>>& blockIndices,
                    const g2o::SparseBlockMatrix<MatrixType>& A) override {
    const int P = upper(A), n = (int)blockIndices.size();
    std::vector<int> r(n), c(n);
    for (int k = 0; k < n; ++k) { r[k] = blockIndices[k].first; c[k] = blockIndices[k].second; }
    inv_.resize(36 * (size_t)n);
    if (!solver_.solvePattern(P, col_ptr_.data(), row_idx_.data(), blocks_.data(), n, r.data(), c.data(), inv_.data()))
      return false;
    for (int k = 0; k < n; ++k)
      std::copy(inv_.begin() + 36 * k, inv_.begin() + 36 * (k + 1), spinv.block(r[k], c[k], true)->data());
    return true;
  }

 private:
  // the upper block CCS of A, as solve() hands it over; returns the number of block columns
  int upper(const g2o::SparseBlockMatrix<MatrixType>& A) {
    const int P = (int)A.blockCols().size();
    col_ptr_.assign(1, 0);
    row_idx_.clear();
    blocks_.clear();
    for (int j = 0; j < P; ++j) {
      for (const auto& rb : A.blockCols()[j]) {
        if (rb.first > j) break;
        row_idx_.push_back(rb.first);
        blocks_.insert(blocks_.end(), rb.second->data(), rb.second->data() + 36);
      }
      col_ptr_.push_back((int)row_idx_.size());
    }
    return P;
  }
  std::vector<double> inv_;
// ---- INTEGRATION.md overrides end

 private:
  svs::LinearSolverBlock6 solver_;
  std::vector<int> col_ptr_, row_idx_;
  std::vector<double> blocks_;
};

int main(int argc, char** argv) {
  if (argc < 3) { printf("usage: chol6_marginals_main in.bin out.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int P = 0, nnzb = 0, n = 0;
  bool ok = fread(&P, 4, 1, f) == 1 && fread(&nnzb, 4, 1, f) == 1 && P > 0 && nnzb > 0;
  std::vector<int> col_ptr(ok ? P + 1 : 0), row_idx(ok ? nnzb : 0);
  std::vector<double> blocks(ok ? 36 * (size_t)nnzb : 0);
  ok = ok && fread(col_ptr.data(), 4, col_ptr.size(), f) == col_ptr.size() && fread(row_idx.data(), 4, row_idx.size(), f) == row_idx.size() &&
       fread(blocks.data(), 8, blocks.size(), f) == blocks.size() && fread(&n, 4, 1, f) == 1 && n >= 0;
  std::vector<int> r(ok ? n : 0), c(ok ? n : 0);
  ok = ok && fread(r.data(), 4, r.size(), f) == r.size() && fread(c.data(), 4, c.size(), f) == c.size();
  fclose(f);
  if (!ok) { printf("BAD_INPUT\n"); return 2; }

  g2o::SparseBlockMatrix<g2o::Matrix6d> A(P);
  for (int j = 0; j < P; ++j)
    for (int k = col_ptr[j]; k < col_ptr[j + 1]; ++k) {
      const int i = row_idx[k];
      const double* src = blocks.data() + 36 * (size_t)k;
      double* up = A.block(i, j, true)->data();
      for (int q = 0; q < 36; ++q) up[q] = src[q];
      if (i != j) {   // the lower mirror: present in the stand-in, never read by the adapter
        double* lo = A.block(j, i, true)->data();
        for (int rr = 0; rr < 6; ++rr)
          for (int cc = 0; cc < 6; ++cc) lo[cc * 6 + rr] = src[rr * 6 + cc];
      }
    }

  std::unique_ptr<g2o::LinearSolver<g2o::Matrix6d>> solver;
  try {
    solver.reset(new LinearSolverSvs<g2o::Matrix6d>());
  } catch (const std::runtime_error& e) {
    printf("NO_GPU %s\n", e.what());
    return 3;
  }
  solver->init();
  double** diag = nullptr;
  const bool ok_blocks = solver->solveBlocks(diag, A);
  std::vector<std::pair<int, int>> idx(n);
  for (int k = 0; k < n; ++k) idx[k] = {r[k], c[k]};
  g2o::SparseBlockMatrix<g2o::MatrixXd> spinv(P);
  const bool ok_pattern = solver->solvePattern(spinv, idx, A);
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  for (int i = 0; i < P; ++i) fwrite(diag[i], 8, 36, o);
  for (int k = 0; k < n; ++k) fwrite(spinv.block(r[k], c[k], false)->data(), 8, 36, o);
  fclose(o);
  for (int i = 0; i < P; ++i) delete[] diag[i];
  delete[] diag;
  printf("OK blocks=%d pattern=%d\n", ok_blocks ? 1 : 0, ok_pattern ? 1 : 0);
  return ok_blocks && ok_pattern ? 0 : 1;
}
