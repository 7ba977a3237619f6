// Host build of TransH's projection (torchkge_b200/csrc/reduce.cuh: the EL_DOT1 sum and transh_project_elem,
// which kge_transh_project and kge_transh_rel_scores are made of) -- test infrastructure.
// tests/test_transh_cpu.py compiles this with g++ (-ffp-contract=off) and compares it, bit for bit, with the
// reference's projection in ATen on the CPU.
#include <stdint.h>

#include "../torchkge_b200/csrc/reduce.cuh"

using namespace kge;

// out[r][k] = projection of ent (one row of dim floats) on the hyperplane of normal norm[r] (n_rel rows)
extern "C" int host_transh_project(int dim, int n_rel, const float* ent, const float* norm, float* out) {
  for (int r = 0; r < n_rel; ++r) {
    const float* w = norm + (size_t)r * dim;
    const float nc = pair_score_natural<EL_DOT1>(dim, ent, ent, w, w);
    for (int k = 0; k < dim; ++k) out[(size_t)r * dim + k] = transh_project_elem(ent[k], nc, w[k]);
  }
  return 0;
}
