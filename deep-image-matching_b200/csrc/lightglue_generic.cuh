// lightglue_generic.cuh - interface of the shape-generic LightGlue (lightglue_generic.cu) used by dimb_lg_* for
// configurations other than descriptor_dim 256 / 4 heads (e.g. the LighterGlue checkpoint: 96 / 1 head / 6 layers).
#pragma once
#include "common.cuh"

struct dimb_lgx;
int lgx_create(dimb_ctx* ctx, const float* weights, size_t n_floats, const dimb_lg_conf* conf, dimb_lgx** out);
void lgx_destroy(dimb_lgx* g);
// dimb_lg_match_dev for these shapes: P <= max_pairs pairs on device pointers, asynchronous on `st`
int lgx_match_dev(dimb_lgx* g, int P, const dimb_feats_dev* f0, const dimb_feats_dev* f1, int64_t* d_matches, float* d_mscores, int* d_n_matches,
                  int* d_stop_layer, int cap, cudaStream_t st);
