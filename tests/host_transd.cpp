// Host build of TransD's projection (torchkge_b200/csrc/reduce.cuh: the EL_DOT1 sum and transd_project_elem,
// which kge_transd_entity_scalars, kge_transd_project and kge_transd_rel_scores are made of) -- test
// infrastructure.  tests/test_transd_cpu.py compiles this with g++ (-ffp-contract=off) and compares it, bit for
// bit, with the reference's expressions in ATen on the CPU.
#include <stdint.h>

#include "../torchkge_b200/csrc/reduce.cuh"

using namespace kge;

// s[i] = (ent_proj[i] * ent[i]).sum() of n rows of ent_dim floats
extern "C" int host_transd_scalars(int ent_dim, int n, const float* ent, const float* ent_proj, float* s) {
  for (int i = 0; i < n; ++i) {
    const float* e = ent + (size_t)i * ent_dim;
    const float* p = ent_proj + (size_t)i * ent_dim;
    s[i] = pair_score_natural<EL_DOT1>(ent_dim, p, p, e, e);
  }
  return 0;
}

// out[r][j] = projection of ent (one row of ent_dim floats, scalar s) under rel_proj[r] (n_rel rows of rel_dim)
extern "C" int host_transd_project(int rel_dim, int n_rel, const float* ent, float s, const float* rel_proj,
                                   float* out) {
  for (int r = 0; r < n_rel; ++r)
    for (int j = 0; j < rel_dim; ++j)
      out[(size_t)r * rel_dim + j] = transd_project_elem(ent[j], s, rel_proj[(size_t)r * rel_dim + j]);
  return 0;
}
