// Symbolic analysis for the supernodal multifrontal LDL^T (host side, runs once).
//
// Replaces what the reference delegates to the vendor solver's analysis phase
// (MUMPS job=1, reference src/Algorithm/LinearSolvers/IpMumpsSolverInterface.cpp:385-446;
//  SPRAL analyse, IpSpralSolverInterface.cpp:448-508).  Input is exactly what
// SparseSymLinearSolverInterface::InitializeStructure delivers
// (IpSparseSymLinearSolverInterface.hpp:139-144): 1-based triplets, either triangle,
// duplicates allowed (they are summed, as IpTripletToCSRConverter.cpp:154-197 does).
//
// Pipeline: unique lower pattern -> saddle-row pairing (zero-diagonal constraint rows are
// matched to a primal neighbour so a 2x2 pivot is always available inside a supernode) ->
// compressed graph -> METIS nested dissection -> elimination tree -> postorder -> column
// structures -> supernodes (leaf-subtree merge + fundamental + relaxed) -> assembly maps,
// child->parent relative indices, level schedule.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

struct AnalyseOptions {
  int ordering = 0;            // 0 = METIS nested dissection, 1 = natural
  int pair_saddle = 1;         // match zero-diagonal rows with a neighbour (needs values)
  int leaf_k = 32;             // merge whole elimination subtrees of <= leaf_k columns
  double relax_frac = 0.05;    // relaxed amalgamation: tolerated fraction of explicit zeros
  int relax_small = 16;        // always merge a last child when merged k <= relax_small
  int dense_n = 48;            // n <= dense_n: a single dense front, natural order
};

struct Symbolic {
  int n = 0;
  int64_t nnz_in = 0;          // triplets delivered
  int64_t nnz_u = 0;           // unique lower entries
  // permutation: perm[new] = old (0-based); iperm[old] = new
  std::vector<int> perm, iperm;
  // triplet e contributes to unique entry t2u[e]; unique entries are sorted by
  // (permuted col, permuted row) so they are grouped by supernode.
  std::vector<int> t2u;
  // segments for deterministic duplicate summation: triplets sorted by unique entry
  std::vector<int64_t> useg_ptr;   // nnz_u+1
  std::vector<int> useg_src;       // nnz_in triplet indices
  std::vector<int> u_row, u_col;   // ORIGINAL (unpermuted, 0-based) row/col of each unique entry (for scaling)
  std::vector<uint32_t> u_dst;     // (local col << 16 | local row) if f < 65536 else see u_dst64
  std::vector<int64_t> u_dst64;    // local row + local col * f  (always filled)

  int nsn = 0;
  std::vector<int> sn_start;       // nsn+1, permuted column ranges
  std::vector<int> sn_parent;      // nsn, -1 for roots
  std::vector<int> sn_level;       // nsn, leaves = 0
  std::vector<int64_t> rows_ptr;   // nsn+1
  std::vector<int> rows;           // permuted row ids > last col, sorted
  std::vector<int> rel;            // same shape as rows: index in the PARENT front (0..f_p)
  std::vector<int> child_ptr;      // nsn+1
  std::vector<int> child_idx;
  std::vector<int64_t> uent_ptr;   // nsn+1 : unique-entry range per supernode
  std::vector<int64_t> L_off;      // nsn+1 : panel f x k, column-major, ld = f
  std::vector<int64_t> cb_off;     // nsn+1 : r x r, column-major, ld = r
  int nlevels = 0;
  std::vector<int> level_ptr;      // nlevels+1
  std::vector<int> level_sn;       // supernodes sorted by (level, front size desc)

  // statistics (algorithmic work, SURVEY.md section 8d formulas)
  int64_t nnzL = 0;                // sum k(k+1)/2 + k r  (entries of L incl. amalgamation zeros)
  int64_t nnzL_true = 0;           // sum of column counts before amalgamation
  double flops_panel = 0;          // sum k^3/3 + k^2 r
  double flops_schur = 0;          // sum k r (r+1)
  int64_t cb_total = 0;            // sum r^2
  int max_front = 0, max_k = 0;
  int n_pairs = 0, n_saddle = 0;
  double t_order = 0, t_symbolic = 0;  // seconds

  int k(int s) const { return sn_start[s + 1] - sn_start[s]; }
  int r(int s) const { return (int)(rows_ptr[s + 1] - rows_ptr[s]); }
  int f(int s) const { return k(s) + r(s); }
};

// values may be nullptr (then no saddle pairing is done). Returns 0 on success,
// negative on invalid input. err receives a message.
int analyse(int n, int64_t nnz, const int* irn, const int* jcn, const double* vals,
            const AnalyseOptions& opt, Symbolic& S, std::string& err);


// Elimination-tree sharding for multi-GPU runs (SURVEY.md section 8e): cut the supernodal tree into a TOP part
// (owner -1, factorised by rank 0 after the contribution blocks of the cut arrive) and disjoint subtrees that
// are assigned to `world` ranks by decreasing work (LPT).  owner[s] = rank of the subtree containing s, or -1.
// Returns the number of independent subtrees below the cut.
int shard_plan(const Symbolic& S, int world, std::vector<int>& owner);

}  // namespace b200
