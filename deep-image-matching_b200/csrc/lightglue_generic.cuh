// lightglue_generic.cuh - interface of the shape-generic fp32 LightGlue (lightglue_generic.cu) used by dimb_lg_* for
// configurations other than descriptor_dim 256 / 4 heads (e.g. the LighterGlue checkpoint: 96 / 1 head / 6 layers).
#pragma once
#include <cmath>

#include "common.cuh"

struct dimb_lgx;
int lgx_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* conf, dimb_lgx** out);
void lgx_destroy(dimb_lgx* g);
int lgx_match(dimb_lgx* g, int P, const dimb_feats* f0, const dimb_feats* f1, int64_t* matches, float* mscores, int* n_matches,
              int* stop_layer, int cap);
// dimb_lg_match_dev for these shapes: P <= max_pairs pairs on device pointers, asynchronous on `st`, bitwise equal to lgx_match
int lgx_match_dev(dimb_lgx* g, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches, float* d_mscores, int* d_n_matches,
                  int* d_stop_layer, int cap, cudaStream_t st);

// filter_matches (lightglue.py:281-297) of the shape-generic path on the host, from the row / column argmaxes a0 [n0] / a1 [n1] and the
// row maxima b0 [n0] the device wrote: row r matches column c = a0[r] when a1[c] == r and exp(b0[r]) > th.  Matches go out in row
// order as (ind0[r], ind1[c]) with score exp(b0[r]), the first cap of them; returns the full count.  An index outside [0, n1) is no
// match: the arrays come from device memory and are not trusted.
inline int lgx_filter(int n0, int n1, const float* b0, const int* a0, const int* a1, const int* ind0, const int* ind1, float th,
                      int64_t* matches, float* mscores, int cap) {
  int cnt = 0;
  for (int r = 0; r < n0; ++r) {
    const int c = a0[r];
    if (c < 0 || c >= n1 || a1[c] != r) continue;  // mutual
    const float e = std::exp(b0[r]);
    if (!(e > th)) continue;
    if (cnt < cap) {
      matches[2 * cnt] = ind0[r];
      matches[2 * cnt + 1] = ind1[c];
      mscores[cnt] = e;
    }
    ++cnt;
  }
  return cnt;
}
