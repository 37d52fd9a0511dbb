// ba_rules.cuh -- the rules of the BA structure analysis that the host analysis (ba_host.cu, set_problem_impl) and the
// device analysis (ba_structure.cu) must apply identically: track padding, the locality key of the internal landmark
// order, the landmarks per build task and the cost of a task in 32-edge waves.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>

namespace svs {

// Track padding: a track of m >= 2 non-anchor observers lo..hi is completed with zero-weight edges to the np frames of
// lo..hi it skips (the anchor frame is never one of them) when the completed track has at most 8 slots and
// np <= max(1, m / 2).  Returns np (0: leave the track as it is).  The sharded window uses the same rule for the block
// pattern every rank must agree on.
__host__ __device__ inline int track_padding(int m, int lo, int hi, int anchor) {
  if (m < 2) return 0;
  const int span = hi - lo + 1 - ((anchor > lo && anchor < hi) ? 1 : 0);   // frames lo..hi without the anchor
  const int np = span - m;
  return (np > 0 && 1 + span <= 8 && np <= (m / 2 > 1 ? m / 2 : 1)) ? np : 0;
}

// Locality key of a landmark with edges: track shape (self flag, slot count K, first and last observer) inside an
// anchor, so that neighbouring warps of the fused kernel scatter into the same blocks of the reduced system.
// Landmarks without edges get ~0 and go last.
__host__ __device__ inline unsigned long long locality_key(int nself, int K, int first, int last) {
  return ((unsigned long long)(nself ? 0 : 1) << 61) | ((unsigned long long)(K & 0xfffff) << 40) |
         ((unsigned long long)(first & 0xfffff) << 20) | (unsigned long long)(last & 0xfffff);
}

// Landmarks per build task: about eleven tasks per SM, so that the persistent grid's tail stays short while coarser
// tasks flush their accumulators less often; clamped to [4, 32].  SVS_BUILD_CHUNK overrides it (at least 1).
inline int build_chunk(int L, int sms) {
  int chunk = L / (std::max(sms, 1) * 11);
  chunk = chunk < 4 ? 4 : (chunk > 32 ? 32 : chunk);
  if (const char* cs = getenv("SVS_BUILD_CHUNK")) chunk = std::max(1, atoi(cs));
  return chunk;
}

// Cost of a task of `cnt` landmarks with kk edges and KK slots each, in waves of k_build_wave (<= 32 edges, 40 slots,
// 8 landmarks per wave), capped at kMaxWaves.  Tasks run longest first.
constexpr int kMaxWaves = 64;
__host__ __device__ inline int task_waves(int kk, int KK, int cnt) {
  const int a = 32 / (kk > 1 ? kk : 1), b = 40 / (KK > 1 ? KK : 1);
  int nw = a < b ? a : b;
  nw = nw > 8 ? 8 : (nw < 1 ? 1 : nw);
  const int w = (cnt + nw - 1) / nw;
  return w < kMaxWaves ? w : kMaxWaves;
}

}  // namespace svs
