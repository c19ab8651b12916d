// AutoInt training: the attention core of one multi-head self-attention layer across the F fields
// (layers/attention.py:67-125), forward and exact backward.  Everything else in a layer (the Q / K / V
// projections, the output projection and all their gradients) is a dense product over R*F rows and runs on
// the library's dense kernels.  The core itself (one warp per (row, head), P recomputed from the lse, no
// atomics) is csrc/attn_core.cuh, instantiated here without a mask.
#include "../../include/b200reco.h"
#include "attn_core.cuh"

namespace b200 {
namespace {

constexpr int AT_MAX_F = 130;   // the inference engine's envelope (autoint.cu)
constexpr int AT_MAX_D = 64;

int attn_setup(AttnShape& s, int64_t R, int32_t F, int32_t H, int32_t hd, float scale, const char* who) {
  B200_REQUIRE(R >= 0, "%s: row count %lld < 0", who, (long long)R);
  B200_REQUIRE(F >= 2 && F <= AT_MAX_F, "%s: field count %d outside [2, %d]", who, F, AT_MAX_F);
  B200_REQUIRE(H >= 1 && hd >= 1 && H <= AT_MAX_D && hd <= AT_MAX_D && H * hd <= AT_MAX_D,
               "%s: num_heads %d x head size %d outside [1, %d]", who, H, hd, AT_MAX_D);
  B200_REQUIRE(isfinite(scale), "%s: scale is not finite", who);
  s.F = F; s.H = H; s.hd = hd; s.scale = scale;
  s.ld = odd(hd); s.lds = odd(F);
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_autoint_attention_forward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                              const float* V, int64_t ldv, int64_t R, int32_t F, int32_t num_heads,
                                              int32_t head_dim, float scale, float* O, int64_t ldo, float* lse,
                                              void* stream) {
  const char* who = "b200_autoint_attention_forward";
  AttnShape s;
  int rc = attn_setup(s, R, F, num_heads, head_dim, scale, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D, "%s: a row stride is below num_heads x head size %lld",
               who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_forward_kernel<false>, (size_t)attn_warp_floats(s, 3) * sizeof(float), items, stream, who, s,
                     AttnMask{nullptr, 0}, Q, ldq, K, ldk, V, ldv, items, O, ldo, lse);
}

extern "C" int b200_autoint_attention_backward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                               const float* V, int64_t ldv, const float* O, int64_t ldo,
                                               const float* lse, const float* dO, int64_t lddo, int64_t R, int32_t F,
                                               int32_t num_heads, int32_t head_dim, float scale, float* dQ, float* dK,
                                               float* dV, int64_t ldg, void* stream) {
  const char* who = "b200_autoint_attention_backward";
  AttnShape s;
  int rc = attn_setup(s, R, F, num_heads, head_dim, scale, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse && dO && dQ && dK && dV, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D && lddo >= D && ldg >= D,
               "%s: a row stride is below num_heads x head size %lld", who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_backward_kernel<false>, (size_t)attn_warp_floats(s, 6) * sizeof(float), items, stream, who, s,
                     AttnMask{nullptr, 0}, Q, ldq, K, ldk, V, ldv, O, ldo, lse, dO, lddo, items, dQ, dK, dV, ldg);
}
