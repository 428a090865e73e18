// GAT's dropout masks (model/gat.py:149-163) drawn on the device from a key: the rule of
// include/lanczosnet_b200.h ("GAT dropout masks").  Element i of the per-channel tensor of a site is kept
// iff word (i & 3) of Philox4x32-10 at counter (i >> 2, site, ctr lo, ctr hi) and key (seed lo, seed hi) is
// >= thr = floor(p * 2^32); a kept value is scaled by s = 1 / (1 - p).  site = (t << 16) | (c << 2) | sigma.
#pragma once
#include "common.cuh"
#include "philox.cuh"

namespace lnb {

enum { GAT_SITE_INPUT = 0, GAT_SITE_ATT = 1, GAT_SITE_WH = 2 };

struct GatDrop {
  const int64_t* key;         // (seed, ctr), device memory
  unsigned long long thr;     // floor(p * 2^32); 2^32 at p = 1 drops everything
  float scale;                // (float)(1 / (1 - p))
  int layer;                  // t
};

// the key words, read once per thread from device memory
struct GatDropKey {
  uint32_t k0, k1, c2, c3;
};

__device__ __forceinline__ GatDropKey gat_drop_key(const GatDrop& d) {
  const uint64_t seed = (uint64_t)d.key[0], ctr = (uint64_t)d.key[1];
  return {(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)ctr, (uint32_t)(ctr >> 32)};
}

__device__ __forceinline__ uint32_t gat_site(int t, int c, int sigma) {
  return ((uint32_t)t << 16) | ((uint32_t)c << 2) | (uint32_t)sigma;
}

// the four words of elements 4q .. 4q+3 of a site
__device__ __forceinline__ uint4 gat_drop_words(const GatDropKey& k, uint64_t q, uint32_t site) {
  return philox4x32_10(make_uint4((uint32_t)q, site, k.c2, k.c3), k.k0, k.k1);
}

__device__ __forceinline__ uint32_t gat_word(const uint4& w, int j) {
  return j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w;
}

__device__ __forceinline__ float gat_drop(float x, uint32_t word, const GatDrop& d) {
  return (unsigned long long)word >= d.thr ? x * d.scale : 0.f;
}

__device__ __forceinline__ float4 gat_drop4(float4 x, const uint4& w, const GatDrop& d) {
  return make_float4(gat_drop(x.x, w.x, d), gat_drop(x.y, w.y, d), gat_drop(x.z, w.z, d), gat_drop(x.w, w.w, d));
}

}  // namespace lnb

// host side: the draw parameters of p in [0, 1], computed in fp64 as the header states
inline lnb::GatDrop gat_drop_params(const int64_t* key, double p, int t) {
  lnb::GatDrop d;
  d.key = key;
  d.thr = (unsigned long long)floor(p * 4294967296.0);
  d.scale = (float)(1.0 / (1.0 - p));
  d.layer = t;
  return d;
}
