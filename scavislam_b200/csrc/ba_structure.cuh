// ba_structure.cuh -- structure analysis of a BA window on the device (ba_structure.cu), for a problem whose arrays
// already lie in device memory (svs_ba_set_problem_device, svs_ba_set_problem_from_map).  It produces the same internal
// layout as the host analysis of set_problem_impl (ba_host.cu): landmarks ordered by (anchor, locality key, caller
// index), edges per landmark with the self edge first and the observers by ascending pose, zero-weight padding edges,
// the build work lists and the co-visibility pattern of the reduced camera system.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace svs {

// error bits of StructHdr::err
enum : int { kStructEdgeRange = 1, kStructPairRange = 2, kStructAnchor = 4, kStructDuplicate = 8 };

// what the host reads back after the analysis (with the pattern bitset and the fixed flags behind it)
struct StructHdr {
  int err;        // kStruct* bits
  int diff;       // 0: the index arrays equal the last structure's (StructIn::k_*); nothing else was computed
  int ne, ns;     // internal edges (with padding), slots
  int Kmax, Kmax_gen;
  int ntasks, ngen, nlong;
};

struct StructIn {
  int P, L, E, C;
  int chunk;   // build_chunk()
  int pad;     // complete tracks with zero-weight edges (track_padding)
  const int* e_point; const int* e_pose; const int* e_anchor; const int* c_i; const int* c_j;
  const unsigned char* fixed;   // may be null (no pose fixed)
  const double* psi;            // [L][3] caller's order
  // the index arrays of the last structure set from device arrays (kept by the handle); compare = 0: none to compare
  int compare;
  const int* k_epoint; const int* k_epose; const int* k_eanchor; const int* k_ci; const int* k_cj;
  const unsigned char* k_fixed;
};

// the analysis' results in device scratch, internal order
struct StructOut {
  StructHdr* hdr;        // hdr | adj | fixed lie at the start of the scratch: one device-to-host copy
  unsigned* adj;         // [P][(P + 31) / 32] co-visibility pattern (tracks and pose-pose constraints)
  unsigned char* fixed;  // [P]
  size_t readback_bytes;
  int *lm_eptr, *lm_sptr, *lm_anchor, *lm_user, *e_pose, *edge_src, *task_lm, *task_cnt, *gen_lm, *long_lm;
  unsigned char* lm_self;
  unsigned char* cls;    // per internal landmark: the work-list class bits (ba_structure.cu)
  double* psi;           // [L][3] internal order
};

// Lays the scratch out at `scratch` and enqueues the analysis on `st`.  With scratch == nullptr nothing is enqueued and
// the bytes the scratch needs are returned; otherwise returns 0 and fills *out.
size_t launch_structure(const StructIn& in, void* scratch, StructOut* out, cudaStream_t st);
// col_need[pos[p]] += the tasks whose slot list holds pose p, and the pose-pose constraints on it (col_need zeroed first)
void launch_col_need(const StructOut& o, int L, int C, const int* c_i, const int* c_j, const int* pos, int* col_need,
                     cudaStream_t st);
// out[li] = psi[lm_user[li]] (3 doubles each)
void launch_psi_gather(const double* psi, const int* lm_user, int L, double* out, cudaStream_t st);

// up to kMaxCopies device-to-device copies in one launch
constexpr int kMaxCopies = 32;
struct CopyJob { const void* src; void* dst; size_t bytes; };
struct CopyList { CopyJob j[kMaxCopies]; int n = 0; void add(const void* s, void* d, size_t b) { if (b) j[n++] = {s, d, b}; } };
void launch_copies(const CopyList& c, cudaStream_t st);

}  // namespace svs
