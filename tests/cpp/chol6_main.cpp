// The g2o linear-solver adapter of INTEGRATION.md §1 against a minimal stand-in for the parts of g2o it touches
// (Matrix6d, SparseBlockMatrix::blockCols(), LinearSolver).  Reads a system written by tests/test_chol6_gpu.py:
//   int32 P, int32 nnzb, int32 col_ptr[P + 1], int32 row_idx[nnzb], float64 blocks[nnzb][36] (column-major),
//   float64 b[6P]
// builds a SparseBlockMatrix holding every block of A (the adapter must skip the lower ones), solves through the
// adapter and writes x[6P].  Exit 0 on success, 1 if not positive definite, 2 on bad input, 3 without a GPU.
#include <cstdio>
#include <map>
#include <memory>
#include <stdexcept>
#include <vector>

#include "svs_b200.hpp"

namespace g2o {
struct Matrix6d {   // Eigen::Matrix<double, 6, 6>: column-major storage
  enum { RowsAtCompileTime = 6, ColsAtCompileTime = 6 };
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
};
}  // namespace g2o

// ---- INTEGRATION.md adapter begin
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

 private:
  svs::LinearSolverBlock6 solver_;
  std::vector<int> col_ptr_, row_idx_;
  std::vector<double> blocks_;
};
// ---- INTEGRATION.md adapter end

int main(int argc, char** argv) {
  if (argc < 3) { printf("usage: chol6_main in.bin out.bin\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int P = 0, nnzb = 0;
  bool ok = fread(&P, 4, 1, f) == 1 && fread(&nnzb, 4, 1, f) == 1 && P > 0 && nnzb > 0;
  std::vector<int> col_ptr(ok ? P + 1 : 0), row_idx(ok ? nnzb : 0);
  std::vector<double> blocks(ok ? 36 * (size_t)nnzb : 0), b(ok ? 6 * (size_t)P : 0), x(b.size(), 0.);
  ok = ok && fread(col_ptr.data(), 4, col_ptr.size(), f) == col_ptr.size() && fread(row_idx.data(), 4, row_idx.size(), f) == row_idx.size() &&
       fread(blocks.data(), 8, blocks.size(), f) == blocks.size() && fread(b.data(), 8, b.size(), f) == b.size();
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
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) lo[c * 6 + r] = src[r * 6 + c];
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
  bool solved = false;
  for (int rep = 0; rep < 2; ++rep) solved = solver->solve(A, x.data(), b.data());   // the second call reuses the analysis
  FILE* o = fopen(argv[2], "wb");
  if (!o) return 2;
  fwrite(x.data(), 8, x.size(), o);
  fclose(o);
  printf("OK solved=%d\n", solved ? 1 : 0);
  return solved ? 0 : 1;
}
