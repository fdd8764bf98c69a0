// fstore.cuh - block layout of the device feature store (dimb_fstore), shared by fstore.cu and the kernels that write slots
// directly (tiles.cu).
#pragma once
#include <vector>

#include "common.cuh"

constexpr int kHdrInts = 8;  // n, H, W, valid, 4 spare

struct SlotPtrs {
  int* hdr;
  __half *kpts, *scores, *tile, *desc;
};

struct dimb_fstore {
  std::vector<void*> mem;
  dimb_ctx* ctx;
  int n_slots, cap, D;
  size_t slot_bytes, off_kpts, off_scores, off_tile, off_desc;
  uint8_t* base = nullptr;
  float *st_k = nullptr, *st_s = nullptr, *st_t = nullptr, *st_d = nullptr;  // staging of the host put
  std::vector<uint8_t> host;  // staging of the host get
};

// The store's geometry by value, for kernels that address any slot.
struct FsLayout {
  uint8_t* base;
  size_t slot_bytes, off_kpts, off_scores, off_tile, off_desc;
  int cap, D;
  __host__ __device__ SlotPtrs at(int slot) const {
    uint8_t* b = base + static_cast<size_t>(slot) * slot_bytes;
    return {reinterpret_cast<int*>(b), reinterpret_cast<__half*>(b + off_kpts), reinterpret_cast<__half*>(b + off_scores),
            reinterpret_cast<__half*>(b + off_tile), reinterpret_cast<__half*>(b + off_desc)};
  }
};

inline FsLayout fs_layout(const dimb_fstore* fs) {
  return {fs->base, fs->slot_bytes, fs->off_kpts, fs->off_scores, fs->off_tile, fs->off_desc, fs->cap, fs->D};
}
