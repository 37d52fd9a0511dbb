// ba_structure.cu -- structure analysis of a BA window whose arrays lie on the device (see ba_structure.cuh).
//
// The passes, all on the handle's stream:
//   validate   range checks of the edges and pose-pose constraints, edges per landmark, first edge of each landmark
//   edge sort  radix sort of the edges by (landmark, not-self, pose): the self edge first, then ascending pose.  Two
//              edges of one landmark in one frame are an error, so this order is total
//   landmarks  anchor, self count, slot count K, padding and locality key per landmark; anchor / duplicate errors
//   order      two stable radix passes: by key (caller index breaks ties), then by anchor bucket
//   emit       lm_eptr / lm_sptr by scan; e_pose, edge_src (with -1 padding edges), lm_anchor, lm_self, lm_user, psi
//   classify   generic / long / run landmarks; runs of identical slot lists, cut every `chunk` landmarks
//   tasks      select, count, stable sort by 32-edge waves (descending)
//   pattern    co-visibility bitset from one landmark per task, the generic and long landmarks and the constraints
// Every kernel after `validate` returns at once when an error was found or the index arrays equal the last
// structure's (StructHdr::diff == 0): the host then reads only the header.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "ba_rules.cuh"
#include "ba_structure.cuh"
#include "ba_types.cuh"
#include "handle.cuh"

namespace svs {
namespace {

constexpr int kThreads = 256;
inline int blocks(long long n) { return (int)std::max<long long>(1, (n + kThreads - 1) / kThreads); }
inline int bits_for(long long v) { int b = 1; while (b < 63 && (1ll << b) <= v) ++b; return b; }   // bits that hold 0..v

// class bits of StructOut::cls
constexpr unsigned char kRunLm = 1, kRunStart = 2, kGeneric = 4, kLong = 8, kTaskHead = 16;

__device__ __forceinline__ bool skip(const StructHdr* h) { return h->err != 0 || h->diff == 0; }

__global__ void k_init(StructHdr* h, int diff) {
  h->err = 0; h->diff = diff; h->ne = 0; h->ns = 0; h->Kmax = 1; h->Kmax_gen = 1; h->ntasks = 0; h->ngen = 0; h->nlong = 0;
}

// same-structure test against the handle's copy of the last device structure
__global__ void k_compare(StructIn in, StructHdr* h) {
  const int n = max(max(in.E, in.C), in.P);
  bool d = false;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < in.E) d |= in.e_point[i] != in.k_epoint[i] || in.e_pose[i] != in.k_epose[i] || in.e_anchor[i] != in.k_eanchor[i];
    if (i < in.C) d |= in.c_i[i] != in.k_ci[i] || in.c_j[i] != in.k_cj[i];
    if (i < in.P) d |= (in.fixed ? in.fixed[i] : 0) != in.k_fixed[i];
  }
  if (d) h->diff = 1;
}

__global__ void k_validate(StructIn in, StructHdr* h, int* cnt, int* first, unsigned char* fixed_out) {
  const int n = max(max(in.E, in.C), in.P);
  const bool work = h->diff != 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < in.P) fixed_out[i] = in.fixed ? in.fixed[i] : 0;
    if (!work) continue;
    if (i < in.E) {
      const int l = in.e_point[i], p = in.e_pose[i], a = in.e_anchor[i];
      if (l < 0 || l >= in.L || p < 0 || p >= in.P || a < 0 || a >= in.P) atomicOr(&h->err, kStructEdgeRange);
      else { atomicAdd(cnt + l, 1); atomicMin(first + l, i); }
    }
    if (i < in.C) {
      const int a = in.c_i[i], b = in.c_j[i];
      if (a < 0 || a >= in.P || b < 0 || b >= in.P || a == b) atomicOr(&h->err, kStructPairRange);
    }
  }
}

// (landmark, not-self, pose); "self" is judged against the anchor of the landmark's first edge in the caller's order,
// as the host analysis does
__global__ void k_edge_keys(StructIn in, const StructHdr* h, const int* first, int pbits, unsigned long long* key, int* val) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= in.E || skip(h)) return;
  const int l = in.e_point[e], p = in.e_pose[e];
  const int anchor = in.e_anchor[first[l]];
  key[e] = ((unsigned long long)l << (pbits + 1)) | ((unsigned long long)(p != anchor) << pbits) | (unsigned long long)p;
  val[e] = e;
}

struct LmInfo {   // per landmark, the caller's order
  int* anchor; int* nself; int* K; int* npad; int* ne; int* bucket; unsigned long long* key;
};

__global__ void k_landmarks(StructIn in, StructHdr* h, const int* eptr, const int* eord, const int* first, LmInfo o) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= in.L || skip(h)) return;
  const int b = eptr[l], en = eptr[l + 1];
  if (b == en) {
    o.anchor[l] = -1; o.nself[l] = 0; o.K[l] = 0; o.npad[l] = 0; o.ne[l] = 0; o.bucket[l] = in.P; o.key[l] = ~0ull;
    return;
  }
  const int anchor = in.e_anchor[first[l]];
  int nself = 0, err = 0, prev = -1;
  for (int k = b; k < en; ++k) {
    const int e = eord[k], p = in.e_pose[e];
    if (in.e_anchor[e] != anchor) err |= kStructAnchor;
    if (p == anchor) ++nself;
    if (k > b && p == prev) err |= kStructDuplicate;
    prev = p;
  }
  if (err) { atomicOr(&h->err, err); return; }
  const int m = (en - b) - nself;
  int K = 1 + m, np = 0;
  if (in.pad && nself <= 1 && m >= 2) {
    np = track_padding(m, in.e_pose[eord[b + nself]], in.e_pose[eord[en - 1]], anchor);
    K += np;
  }
  atomicMax(&h->Kmax, K);
  const int fi = b + (nself ? 1 : 0) < en ? b + (nself ? 1 : 0) : b;
  o.anchor[l] = anchor; o.nself[l] = nself; o.K[l] = K; o.npad[l] = np; o.ne[l] = (en - b) + np; o.bucket[l] = anchor;
  o.key[l] = locality_key(nself, K, in.e_pose[eord[fi]], in.e_pose[eord[en - 1]]);
}

__global__ void k_iota(int n, int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}

__global__ void k_bucket_of(int L, const StructHdr* h, const int* ord, const int* bucket, int* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L || skip(h)) return;
  out[i] = bucket[ord[i]];
}

__global__ void k_counts(int L, const StructHdr* h, const int* order, LmInfo o, int* cnt_e, int* cnt_s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > L || skip(h)) return;
  cnt_e[i] = i < L ? o.ne[order[i]] : 0;
  cnt_s[i] = i < L ? o.K[order[i]] : 0;
}

// internal landmark li: its edges (the completed track's frames lo..hi with -1 for a padding edge), anchor, self flag,
// caller index and psi
__global__ void k_emit(StructIn in, const StructHdr* h, const int* order, const int* eptr, const int* eord, LmInfo o,
                       StructOut out) {
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  if (li >= in.L || skip(h)) return;
  const int l = order[li];
  out.lm_user[li] = l;
  for (int q = 0; q < 3; ++q) out.psi[3 * (size_t)li + q] = in.psi[3 * (size_t)l + q];
  const int anchor = o.anchor[l];
  out.lm_anchor[li] = anchor < 0 ? 0 : anchor;
  out.lm_self[li] = (unsigned char)o.nself[l];
  if (anchor < 0) return;
  int at = out.lm_eptr[li], k = eptr[l];
  const int en = eptr[l + 1];
  if (o.npad[l] == 0) {
    for (; k < en; ++k, ++at) { const int e = eord[k]; out.e_pose[at] = in.e_pose[e]; out.edge_src[at] = e; }
    return;
  }
  if (o.nself[l]) { out.e_pose[at] = anchor; out.edge_src[at++] = eord[k++]; }
  const int lo = in.e_pose[eord[k]], hi = in.e_pose[eord[en - 1]];
  for (int p = lo; p <= hi; ++p) {
    if (p == anchor) continue;
    out.e_pose[at] = p;
    if (k < en && in.e_pose[eord[k]] == p) out.edge_src[at++] = eord[k++];
    else out.edge_src[at++] = -1;
  }
}

__device__ __forceinline__ bool same_slots(const StructOut& o, int la, int lb) {
  const int b0 = o.lm_eptr[la], b1 = o.lm_eptr[lb], ka = o.lm_eptr[la + 1] - b0;
  if (ka != o.lm_eptr[lb + 1] - b1 || o.lm_anchor[la] != o.lm_anchor[lb] || o.lm_self[la] != o.lm_self[lb]) return false;
  for (int i = 0; i < ka; ++i)
    if (o.e_pose[b0 + i] != o.e_pose[b1 + i]) return false;
  return true;
}

__device__ __forceinline__ bool run_landmark(const StructOut& o, int li) {
  const int kk = o.lm_eptr[li + 1] - o.lm_eptr[li], KK = o.lm_sptr[li + 1] - o.lm_sptr[li];
  return kk > 0 && KK <= 8;
}

// work-list class of each internal landmark; run_start[li] = li at the first landmark of a run, else -1
__global__ void k_classify(int L, StructHdr* h, StructOut o, int* run_start) {
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  if (li >= L || skip(h)) return;
  if (li == L - 1) { h->ne = o.lm_eptr[L]; h->ns = o.lm_sptr[L]; }
  const int kk = o.lm_eptr[li + 1] - o.lm_eptr[li], KK = o.lm_sptr[li + 1] - o.lm_sptr[li];
  unsigned char c;
  if (kk > 0 && KK > kMaxTrack) c = kLong;
  else if (kk == 0 || KK > 8) { c = kGeneric; atomicMax(&h->Kmax_gen, KK); }
  else c = (li > 0 && run_landmark(o, li - 1) && same_slots(o, li - 1, li)) ? kRunLm : (kRunLm | kRunStart);
  o.cls[li] = c;
  run_start[li] = (c & kRunStart) ? li : -1;
}

// a task starts at every chunk-th landmark of a run (run_first = the run's first landmark, by a max-scan)
__global__ void k_heads(int L, int chunk, const StructHdr* h, StructOut o, const int* run_first, unsigned char* f_task,
                        unsigned char* f_gen, unsigned char* f_long) {
  const int li = blockIdx.x * blockDim.x + threadIdx.x;
  if (li >= L || skip(h)) return;
  unsigned char c = o.cls[li];
  if ((c & kRunLm) && (li - run_first[li]) % chunk == 0) c |= kTaskHead;
  o.cls[li] = c;
  f_task[li] = (c & kTaskHead) != 0;
  f_gen[li] = (c & kGeneric) != 0;
  f_long[li] = (c & kLong) != 0;
}

// landmarks of each task and its sort key (kMaxWaves - waves: the longest first); entries past ntasks sort last
__global__ void k_task_cnt(int L, int chunk, const StructHdr* h, const StructOut o, const int* task_lm0, int* cnt0,
                           unsigned char* wkey, int* tid) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= L || skip(h)) return;
  tid[t] = t;
  if (t >= h->ntasks) { wkey[t] = 255; return; }
  const int li = task_lm0[t];
  int c = 1;
  while (c < chunk && li + c < L && (o.cls[li + c] & (kRunLm | kRunStart)) == kRunLm) ++c;
  cnt0[t] = c;
  const int kk = o.lm_eptr[li + 1] - o.lm_eptr[li], KK = o.lm_sptr[li + 1] - o.lm_sptr[li];
  wkey[t] = (unsigned char)(kMaxWaves - task_waves(kk, KK, c));
}

__global__ void k_task_gather(int L, const StructHdr* h, const int* perm, const int* task_lm0, const int* cnt0, StructOut o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L || skip(h) || i >= h->ntasks) return;
  o.task_lm[i] = task_lm0[perm[i]];
  o.task_cnt[i] = cnt0[perm[i]];
}

__device__ __forceinline__ void set_pair(unsigned* adj, int W, int a, int b) {
  atomicOr(adj + (size_t)a * W + (b >> 5), 1u << (b & 31));
  atomicOr(adj + (size_t)b * W + (a >> 5), 1u << (a & 31));
}

// all pairs inside a track (anchor and every slot after the self edge) of one landmark per task, of every generic
// landmark with edges and every long landmark; the pose-pose constraints
__global__ void k_pattern(int L, int C, int P, const StructHdr* h, StructOut o, const int* c_i, const int* c_j) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L + C || skip(h)) return;
  const int W = (P + 31) / 32;
  if (i >= L) { set_pair(o.adj, W, c_i[i - L], c_j[i - L]); return; }
  const unsigned char c = o.cls[i];
  const int b = o.lm_eptr[i] + o.lm_self[i], en = o.lm_eptr[i + 1], a = o.lm_anchor[i];
  if (!((c & kTaskHead) || (c & kLong) || ((c & kGeneric) && en > o.lm_eptr[i]))) return;
  for (int x = b; x < en; ++x) {
    const int px = o.e_pose[x];
    set_pair(o.adj, W, a, px);
    for (int y = x + 1; y < en; ++y) set_pair(o.adj, W, px, o.e_pose[y]);
  }
}

__global__ void k_col_need(int L, int C, StructOut o, const int* c_i, const int* c_j, const int* pos, int* col_need) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L + C) return;
  if (i >= L) { atomicAdd(col_need + pos[c_i[i - L]], 1); atomicAdd(col_need + pos[c_j[i - L]], 1); return; }
  if (!(o.cls[i] & kTaskHead)) return;
  atomicAdd(col_need + pos[o.lm_anchor[i]], 1);
  for (int x = o.lm_eptr[i] + o.lm_self[i]; x < o.lm_eptr[i + 1]; ++x) atomicAdd(col_need + pos[o.e_pose[x]], 1);
}

__global__ void k_psi_gather(const double* psi, const int* lm_user, int L, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * L) return;
  out[i] = psi[3 * (size_t)lm_user[i / 3] + i % 3];
}

// blockIdx.y = job; 16-byte words where both ends are 16-byte aligned, else bytes
__global__ void k_copies(CopyList c) {
  const CopyJob j = c.j[blockIdx.y];
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const char* s = static_cast<const char*>(j.src);
  char* d = static_cast<char*>(j.dst);
  size_t done = 0;
  if ((((size_t)s | (size_t)d) & 15) == 0) {
    const size_t n16 = j.bytes / 16;
    for (size_t i = tid; i < n16; i += stride) reinterpret_cast<int4*>(d)[i] = reinterpret_cast<const int4*>(s)[i];
    done = n16 * 16;
  }
  for (size_t i = done + tid; i < j.bytes; i += stride) d[i] = s[i];
}

}  // namespace

size_t launch_structure(const StructIn& in, void* scratch, StructOut* out, cudaStream_t st) {
  const int P = in.P, L = in.L, E = in.E, C = in.C;
  const int W = (P + 31) / 32;
  Bump m{static_cast<char*>(scratch)};
  StructOut o{};
  o.hdr = m.take<StructHdr>(1);
  o.adj = m.take<unsigned>((size_t)P * W);
  o.fixed = m.take<unsigned char>(P);
  o.readback_bytes = m.off;
  int* cnt = m.take<int>((size_t)L + 1);
  int* first = m.take<int>(L);
  int* eptr = m.take<int>((size_t)L + 1);
  unsigned long long* ekey = m.take<unsigned long long>(E);
  unsigned long long* ekey2 = m.take<unsigned long long>(E);
  int* eval = m.take<int>(E);
  int* eord = m.take<int>(E);
  LmInfo li{m.take<int>(L), m.take<int>(L), m.take<int>(L), m.take<int>(L), m.take<int>(L), m.take<int>(L),
            m.take<unsigned long long>(L)};
  unsigned long long* lkey2 = m.take<unsigned long long>(L);
  int* iota = m.take<int>(L);
  int* ord1 = m.take<int>(L);
  int* bkt = m.take<int>(L);
  int* bkt2 = m.take<int>(L);
  int* order = m.take<int>(L);
  int* cnt_e = m.take<int>((size_t)L + 1);
  int* cnt_s = m.take<int>((size_t)L + 1);
  const size_t ne_max = 2 * (size_t)E;   // a completed track at most doubles its observer edges
  o.lm_eptr = m.take<int>((size_t)L + 1); o.lm_sptr = m.take<int>((size_t)L + 1);
  o.lm_anchor = m.take<int>(L); o.lm_user = m.take<int>(L); o.lm_self = m.take<unsigned char>(L);
  o.psi = m.take<double>(3 * (size_t)L);
  o.e_pose = m.take<int>(ne_max); o.edge_src = m.take<int>(ne_max);
  o.cls = m.take<unsigned char>(L);
  int* run_start = m.take<int>(L);
  int* run_first = m.take<int>(L);
  unsigned char* f_task = m.take<unsigned char>(L);
  unsigned char* f_gen = m.take<unsigned char>(L);
  unsigned char* f_long = m.take<unsigned char>(L);
  int* task_lm0 = m.take<int>(L);
  int* cnt0 = m.take<int>(L);
  unsigned char* wkey = m.take<unsigned char>(L);
  unsigned char* wkey2 = m.take<unsigned char>(L);
  int* tid = m.take<int>(L);
  int* tperm = m.take<int>(L);
  o.task_lm = m.take<int>(L); o.task_cnt = m.take<int>(L); o.gen_lm = m.take<int>(L); o.long_lm = m.take<int>(L);

  const int pbits = bits_for(std::max(P - 1, 0)), lbits = bits_for(std::max(L - 1, 0)), bbits = bits_for(P);
  const int ebits = std::min(64, lbits + 1 + pbits);
  thrust::counting_iterator<int> count0(0);
  // CUB's temporary storage: the largest of the calls below (sized in the sizing pass)
  size_t tmp = 0;
  auto need = [&](size_t b) { tmp = std::max(tmp, b); };
  {
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, cnt, eptr, L + 1); need(b);
    cub::DeviceRadixSort::SortPairs(nullptr, b, ekey, ekey2, eval, eord, E, 0, ebits); need(b);
    cub::DeviceRadixSort::SortPairs(nullptr, b, li.key, lkey2, iota, ord1, L, 0, 64); need(b);
    cub::DeviceRadixSort::SortPairs(nullptr, b, bkt, bkt2, ord1, order, L, 0, bbits); need(b);
    cub::DeviceScan::InclusiveScan(nullptr, b, run_start, run_first, cub::Max(), L); need(b);
    cub::DeviceSelect::Flagged(nullptr, b, count0, f_task, task_lm0, &o.hdr->ntasks, L); need(b);
    cub::DeviceRadixSort::SortPairs(nullptr, b, wkey, wkey2, tid, tperm, L, 0, 8); need(b);
  }
  void* ctmp = m.take<char>(tmp);
  if (!scratch) return m.off;

  const int nmax = std::max(std::max(E, C), P);
  k_init<<<1, 1, 0, st>>>(o.hdr, in.compare ? 0 : 1);
  cudaMemsetAsync(o.adj, 0, sizeof(unsigned) * (size_t)P * W, st);
  cudaMemsetAsync(cnt, 0, sizeof(int) * ((size_t)L + 1), st);
  cudaMemsetAsync(first, 0x7f, sizeof(int) * (size_t)std::max(L, 1), st);
  if (in.compare && nmax) k_compare<<<std::min(blocks(nmax), 1024), kThreads, 0, st>>>(in, o.hdr);
  if (nmax) k_validate<<<std::min(blocks(nmax), 2048), kThreads, 0, st>>>(in, o.hdr, cnt, first, o.fixed);
  cub::DeviceScan::ExclusiveSum(ctmp, tmp, cnt, eptr, L + 1, st);
  if (E) {
    k_edge_keys<<<blocks(E), kThreads, 0, st>>>(in, o.hdr, first, pbits, ekey, eval);
    cub::DeviceRadixSort::SortPairs(ctmp, tmp, ekey, ekey2, eval, eord, E, 0, ebits, st);
  }
  if (L) {
    k_landmarks<<<blocks(L), kThreads, 0, st>>>(in, o.hdr, eptr, eord, first, li);
    k_iota<<<blocks(L), kThreads, 0, st>>>(L, iota);
    // internal order: by key, the caller's index breaking ties (stable), then by anchor bucket (stable)
    cub::DeviceRadixSort::SortPairs(ctmp, tmp, li.key, lkey2, iota, ord1, L, 0, 64, st);
    k_bucket_of<<<blocks(L), kThreads, 0, st>>>(L, o.hdr, ord1, li.bucket, bkt);
    cub::DeviceRadixSort::SortPairs(ctmp, tmp, bkt, bkt2, ord1, order, L, 0, bbits, st);
  }
  k_counts<<<blocks((long long)L + 1), kThreads, 0, st>>>(L, o.hdr, order, li, cnt_e, cnt_s);
  cub::DeviceScan::ExclusiveSum(ctmp, tmp, cnt_e, o.lm_eptr, L + 1, st);
  cub::DeviceScan::ExclusiveSum(ctmp, tmp, cnt_s, o.lm_sptr, L + 1, st);
  if (L) {
    k_emit<<<blocks(L), kThreads, 0, st>>>(in, o.hdr, order, eptr, eord, li, o);
    k_classify<<<blocks(L), kThreads, 0, st>>>(L, o.hdr, o, run_start);
    cub::DeviceScan::InclusiveScan(ctmp, tmp, run_start, run_first, cub::Max(), L, st);
    k_heads<<<blocks(L), kThreads, 0, st>>>(L, in.chunk, o.hdr, o, run_first, f_task, f_gen, f_long);
    cub::DeviceSelect::Flagged(ctmp, tmp, count0, f_task, task_lm0, &o.hdr->ntasks, L, st);
    cub::DeviceSelect::Flagged(ctmp, tmp, count0, f_gen, o.gen_lm, &o.hdr->ngen, L, st);
    cub::DeviceSelect::Flagged(ctmp, tmp, count0, f_long, o.long_lm, &o.hdr->nlong, L, st);
    k_task_cnt<<<blocks(L), kThreads, 0, st>>>(L, in.chunk, o.hdr, o, task_lm0, cnt0, wkey, tid);
    cub::DeviceRadixSort::SortPairs(ctmp, tmp, wkey, wkey2, tid, tperm, L, 0, 8, st);
    k_task_gather<<<blocks(L), kThreads, 0, st>>>(L, o.hdr, tperm, task_lm0, cnt0, o);
  }
  if (L + C) k_pattern<<<blocks((long long)L + C), kThreads, 0, st>>>(L, C, P, o.hdr, o, in.c_i, in.c_j);
  *out = o;
  return 0;
}

void launch_col_need(const StructOut& o, int L, int C, const int* c_i, const int* c_j, const int* pos, int* col_need,
                     cudaStream_t st) {
  if (L + C) k_col_need<<<blocks((long long)L + C), kThreads, 0, st>>>(L, C, o, c_i, c_j, pos, col_need);
}

void launch_psi_gather(const double* psi, const int* lm_user, int L, double* out, cudaStream_t st) {
  if (L) k_psi_gather<<<blocks(3ll * L), kThreads, 0, st>>>(psi, lm_user, L, out);
}

void launch_copies(const CopyList& c, cudaStream_t st) {
  if (c.n == 0) return;
  size_t mx = 0;
  for (int i = 0; i < c.n; ++i) mx = std::max(mx, c.j[i].bytes);
  const int bx = (int)std::min<size_t>(std::max<size_t>(1, (mx / 16 + kThreads - 1) / kThreads), 256);
  k_copies<<<dim3(bx, c.n), kThreads, 0, st>>>(c);
}

}  // namespace svs
