// Host-only entry points of the symbolic analysis (no CUDA needed): used by the CPU test-suite
// and by tooling that wants to inspect the elimination tree / supernode partition.
#include <cstring>
#include <string>
#include <vector>

#include "symbolic.hpp"

using namespace b200;

struct SymHandle { Symbolic S; std::string err; };

extern "C" {

/* b200ldlt_symbolic_create with a Schur set: vars[0..m) (0-based) become the last m pivot positions, one root supernode */
void* b200ldlt_symbolic_create_schur(int dim, int nonzeros, const int* irn, const int* jcn, const double* vals,
                                     int ordering, int pair_saddle, int leaf_k, double relax_frac, int m, const int* vars) {
  SymHandle* h = new SymHandle();
  AnalyseOptions ao;
  ao.ordering = ordering; ao.pair_saddle = pair_saddle;
  if (leaf_k > 0) ao.leaf_k = leaf_k;
  if (relax_frac >= 0) ao.relax_frac = relax_frac;
  if (m > 0 && vars) ao.sc_vars.assign(vars, vars + m);
  int rc = analyse(dim, nonzeros, irn, jcn, vals, ao, h->S, h->err);
  if (rc != 0) { fprintf(stderr, "[b200ldlt] symbolic analysis failed: %s\n", h->err.c_str()); delete h; return nullptr; }
  return h;
}

void* b200ldlt_symbolic_create(int dim, int nonzeros, const int* irn, const int* jcn, const double* vals,
                               int ordering, int pair_saddle, int leaf_k, double relax_frac) {
  return b200ldlt_symbolic_create_schur(dim, nonzeros, irn, jcn, vals, ordering, pair_saddle, leaf_k, relax_frac, 0, nullptr);
}

void b200ldlt_symbolic_free(void* p) { delete (SymHandle*)p; }

long long b200ldlt_symbolic_get(void* p, const char* name, long long* out, long long cap) {
  if (!p || !name) return -1;
  const Symbolic& S = ((SymHandle*)p)->S;
  std::string nm(name);
#define RET(vec)                                                                          \
  do {                                                                                    \
    long long len = (long long)(vec).size();                                              \
    if (out) for (long long i = 0; i < len && i < cap; ++i) out[i] = (long long)(vec)[i]; \
    return len;                                                                           \
  } while (0)
  if (nm == "perm") RET(S.perm);
  if (nm == "sn_start") RET(S.sn_start);
  if (nm == "sn_parent") RET(S.sn_parent);
  if (nm == "rows_ptr") RET(S.rows_ptr);
  if (nm == "rows") RET(S.rows);
  if (nm == "rel") RET(S.rel);
  if (nm == "L_off") RET(S.L_off);
  if (nm == "cb_off") RET(S.cb_off);
  if (nm == "u_dst64") RET(S.u_dst64);
  if (nm == "uent_ptr") RET(S.uent_ptr);
  if (nm == "t2u") RET(S.t2u);
  if (nm == "sn_level") RET(S.sn_level);
  if (nm == "level_ptr") RET(S.level_ptr);
  if (nm == "level_sn") RET(S.level_sn);
  if (nm == "child_ptr") RET(S.child_ptr);
  if (nm == "child_idx") RET(S.child_idx);
#undef RET
  if (nm == "stats") {
    // n, nsn, nlevels, max_front, max_k, n_saddle, n_pairs, nnzL, nnzL_true, cb_total, flops_panel, flops_schur, ms_order, ms_symbolic
    long long v[14] = {S.n, S.nsn, S.nlevels, S.max_front, S.max_k, S.n_saddle, S.n_pairs, (long long)S.nnzL,
                       (long long)S.nnzL_true, (long long)S.cb_total, (long long)S.flops_panel, (long long)S.flops_schur,
                       (long long)(S.t_order * 1e3), (long long)(S.t_symbolic * 1e3)};
    if (out) for (int i = 0; i < 14 && i < cap; ++i) out[i] = v[i];
    return 14;
  }
  return -1;
}


/* owner[s] for every supernode (rank of its subtree, -1 = top part); returns the number of subtrees below the cut */
long long b200ldlt_symbolic_shard(void* p, int world, long long* out, long long cap) {
  if (!p) return -1;
  std::vector<int> owner;
  int nsub = shard_plan(((SymHandle*)p)->S, world, owner);
  if (out) for (long long i = 0; i < (long long)owner.size() && i < cap; ++i) out[i] = owner[i];
  return nsub;
}

}  // extern "C"
