// Host symbolic analysis -- see symbolic.hpp for the pipeline and the reference citations.
#include "symbolic.hpp"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <numeric>

// METIS 5.x from the CUDA toolkit's libmetis_static.a (idx_t is 64-bit there; no header is shipped).
extern "C" int METIS_SetDefaultOptions(int64_t* options);
extern "C" int METIS_NodeND(int64_t* nvtxs, int64_t* xadj, int64_t* adjncy, int64_t* vwgt,
                            int64_t* options, int64_t* perm, int64_t* iperm);

namespace b200 {
namespace {

double now_s() {
  using namespace std::chrono;
  return duration<double>(steady_clock::now().time_since_epoch()).count();
}

// Liu's elimination-tree algorithm with path compression, driven from the symmetric
// adjacency structure under the labelling iperm (old->new), perm (new->old).
void etree_from_graph(int n, const std::vector<int64_t>& xadj, const std::vector<int>& adj,
                      const std::vector<int>& perm, const std::vector<int>& iperm,
                      std::vector<int>& parent) {
  parent.assign(n, -1);
  std::vector<int> anc(n, -1);
  for (int k = 0; k < n; ++k) {
    int old = perm[k];
    for (int64_t p = xadj[old]; p < xadj[old + 1]; ++p) {
      int i = iperm[adj[p]];
      while (i != -1 && i < k) {
        int nxt = anc[i];
        anc[i] = k;
        if (nxt == -1) parent[i] = k;
        i = nxt;
      }
    }
  }
}

// Postorder with children visited in ascending label order (keeps a node that directly
// precedes its parent adjacent to it -- needed for saddle pairs).
void postorder(int n, const std::vector<int>& parent, std::vector<int>& post) {
  std::vector<int> head(n, -1), next(n, -1);
  std::vector<int> roots;
  for (int j = n - 1; j >= 0; --j) {  // descending insert => ascending lists
    if (parent[j] < 0) roots.push_back(j);
    else { next[j] = head[parent[j]]; head[parent[j]] = j; }
  }
  std::reverse(roots.begin(), roots.end());
  post.clear();
  post.reserve(n);
  std::vector<int> stack;
  for (int rt : roots) {
    stack.push_back(rt);
    while (!stack.empty()) {
      int v = stack.back();
      int c = head[v];
      if (c >= 0) { head[v] = next[c]; stack.push_back(c); }
      else { post.push_back(v); stack.pop_back(); }
    }
  }
}

// Entries (column c, row r, id) sorted by (c, r, id): two stable counting passes (by r, then by c) over entries given
// in ascending id order -- same result as std::sort on ((c*n + r), id) pairs at a fraction of the time.
struct Ent { int c, r, id; };
void sort_entries(int n, std::vector<Ent>& a) {
  const size_t m = a.size();
  std::vector<Ent> b(m);
  std::vector<int64_t> cnt((size_t)n + 1);
  std::fill(cnt.begin(), cnt.end(), 0);
  for (const Ent& x : a) cnt[x.r + 1]++;
  for (int i = 0; i < n; ++i) cnt[i + 1] += cnt[i];
  for (const Ent& x : a) b[cnt[x.r]++] = x;
  std::fill(cnt.begin(), cnt.end(), 0);
  for (const Ent& x : b) cnt[x.c + 1]++;
  for (int i = 0; i < n; ++i) cnt[i + 1] += cnt[i];
  for (const Ent& x : b) a[cnt[x.c]++] = x;
}

}  // namespace

int analyse(int n, int64_t nnz, const int* irn, const int* jcn, const double* vals,
            const AnalyseOptions& opt, Symbolic& S, std::string& err) {
  double t0 = now_s();
  S = Symbolic();
  S.n = n;
  S.nnz_in = nnz;
  if (n <= 0 || nnz < 0) { err = "analyse: empty system"; return -1; }
  for (int64_t e = 0; e < nnz; ++e) {
    if (irn[e] < 1 || irn[e] > n || jcn[e] < 1 || jcn[e] > n) { err = "analyse: index out of range"; return -2; }
  }
  // Schur variables: is_sc marks them; E (the rest) is ordered and eliminated, S follows in the caller's order
  const std::vector<int>& sc = opt.sc_vars;
  const int m = (int)sc.size();
  std::vector<char> is_sc(n, 0);
  if (m >= n) { err = "analyse: the Schur set must leave a variable to eliminate"; return -2; }
  for (int v : sc) {
    if (v < 0 || v >= n || is_sc[v]) { err = "analyse: Schur variable out of range or repeated"; return -2; }
    is_sc[v] = 1;
  }

  // ---- 1. unique lower pattern in ORIGINAL labels -------------------------------------------
  std::vector<Ent> keyed((size_t)nnz);
  for (int64_t e = 0; e < nnz; ++e) {
    int i = irn[e] - 1, j = jcn[e] - 1;
    keyed[e] = Ent{std::min(i, j), std::max(i, j), (int)e};
  }
  sort_entries(n, keyed);
  std::vector<int> ur, uc;        // original unique entries
  std::vector<double> uv;         // summed values (only if vals)
  std::vector<int> t2u0((size_t)nnz);
  ur.reserve(nnz); uc.reserve(nnz);
  for (int64_t q = 0; q < nnz; ++q) {
    if (q == 0 || keyed[q].c != keyed[q - 1].c || keyed[q].r != keyed[q - 1].r) {
      uc.push_back(keyed[q].c);
      ur.push_back(keyed[q].r);
      if (vals) uv.push_back(0.0);
    }
    t2u0[keyed[q].id] = (int)ur.size() - 1;
    if (vals) uv.back() += vals[keyed[q].id];
  }
  { std::vector<Ent>().swap(keyed); }
  const int64_t nu = (int64_t)ur.size();
  S.nnz_u = nu;

  // ---- 2. symmetric adjacency (no diagonal) ---------------------------------------------------
  std::vector<int64_t> xadj(n + 1, 0);
  for (int64_t u = 0; u < nu; ++u) if (ur[u] != uc[u]) { xadj[ur[u] + 1]++; xadj[uc[u] + 1]++; }
  for (int i = 0; i < n; ++i) xadj[i + 1] += xadj[i];
  std::vector<int> adj((size_t)xadj[n]);
  std::vector<double> adjw;
  if (vals) adjw.resize((size_t)xadj[n]);
  {
    std::vector<int64_t> pos(xadj.begin(), xadj.end() - 1);
    for (int64_t u = 0; u < nu; ++u) if (ur[u] != uc[u]) {
      if (vals) { adjw[pos[ur[u]]] = std::fabs(uv[u]); adjw[pos[uc[u]]] = std::fabs(uv[u]); }
      adj[pos[ur[u]]++] = uc[u];
      adj[pos[uc[u]]++] = ur[u];
    }
  }

  // ---- 3. saddle pairing ----------------------------------------------------------------------
  std::vector<int> partner(n, -1);
  std::vector<char> saddle(n, 0);
  if (vals && opt.pair_saddle) {
    std::vector<double> diag(n, 0.0);
    for (int64_t u = 0; u < nu; ++u) if (ur[u] == uc[u]) diag[ur[u]] = uv[u];
    // saddle row = (numerically) zero diagonal relative to its off-diagonal entries: the constraint block of the
    // KKT system arrives as explicit zeros, or as -delta_c ~ 1e-8 after a regularisation
    // (reference src/Algorithm/IpStdAugSystemSolver.cpp:420-426)
    for (int i = 0; i < n; ++i) {
      double om = 0.0;
      for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p) om = std::max(om, adjw[p]);
      if (std::fabs(diag[i]) <= 1e-7 * om || (diag[i] == 0.0)) { saddle[i] = 1; S.n_saddle++; }
    }
    struct Cand { double w; int s, x; };
    std::vector<Cand> cand;
    for (int i = 0; i < n; ++i) if (saddle[i] && !is_sc[i])
      for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p)
        if (!saddle[adj[p]] && !is_sc[adj[p]] && adjw[p] > 0.0) cand.push_back({adjw[p], i, adj[p]});
    std::sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) {
      if (a.w != b.w) return a.w > b.w;
      if (a.s != b.s) return a.s < b.s;
      return a.x < b.x;
    });
    for (const Cand& c : cand)
      if (partner[c.s] < 0 && partner[c.x] < 0) { partner[c.s] = c.x; partner[c.x] = c.s; S.n_pairs++; }
    // completion with SHORT augmenting paths only.  A maximum-cardinality matching can be numerically poor
    // (on chain-like Jacobians a long alternating path shifts a whole segment onto its weakest entries and
    // the pivot blocks become Kahan-like triangular matrices), so a path is accepted only if it has at most
    // kMaxHops saddle rows and every newly matched edge keeps a decent fraction of its row's largest entry.
    // Saddle rows left unmatched are still eliminated through in-supernode 2x2 pivots where possible.
    const int kMaxHops = 3;
    const double kMinFrac = 0.05;
    std::vector<double> rowmax(n, 0.0);
    for (int i = 0; i < n; ++i) if (saddle[i])
      for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p) rowmax[i] = std::max(rowmax[i], adjw[p]);
    std::vector<int> visit(n, -1), from_s(n, -1), depth(n, 0);
    std::vector<int> queue;
    for (int s0 = 0; s0 < n; ++s0) {
      if (!saddle[s0] || partner[s0] >= 0 || is_sc[s0]) continue;
      queue.clear();
      queue.push_back(s0);
      depth[s0] = 1;
      int found_x = -1;
      for (size_t qh = 0; qh < queue.size() && found_x < 0; ++qh) {
        int sq = queue[qh];
        for (int64_t p = xadj[sq]; p < xadj[sq + 1]; ++p) {
          int x = adj[p];
          if (saddle[x] || is_sc[x] || visit[x] == s0) continue;
          if (!(adjw[p] >= kMinFrac * rowmax[sq]) || !(adjw[p] > 0.0)) continue;
          visit[x] = s0;
          from_s[x] = sq;
          if (partner[x] < 0) { found_x = x; break; }
          int s2 = partner[x];
          if (depth[sq] < kMaxHops) { depth[s2] = depth[sq] + 1; queue.push_back(s2); }
        }
      }
      if (found_x >= 0) {
        int x = found_x;
        while (true) {
          int sq = from_s[x];
          int prev_x = partner[sq];
          partner[sq] = x; partner[x] = sq;
          if (sq == s0) break;
          x = prev_x;
        }
        S.n_pairs++;
      }
    }
  }

  // ---- 4. compressed graph --------------------------------------------------------------------
  std::vector<int> cnode(n, -1);
  std::vector<int> cfirst, csecond;  // members: primal first, saddle second (or -1)
  for (int i = 0; i < n; ++i) {
    if (cnode[i] >= 0 || is_sc[i]) continue;
    if (partner[i] < 0) { cnode[i] = (int)cfirst.size(); cfirst.push_back(i); csecond.push_back(-1); }
    else {
      int x = saddle[i] ? partner[i] : i, c = saddle[i] ? i : partner[i];
      cnode[x] = cnode[c] = (int)cfirst.size();
      cfirst.push_back(x); csecond.push_back(c);
    }
  }
  const int nce = (int)cfirst.size();    // the nodes of E: the ordering sees these only
  for (int v : sc) { cnode[v] = (int)cfirst.size(); cfirst.push_back(v); csecond.push_back(-1); }
  const int nc = (int)cfirst.size();
  std::vector<int> cperm(nc);
  std::iota(cperm.begin(), cperm.end(), 0);
  double t_ord0 = now_s();
  if (opt.ordering == 0 && n > opt.dense_n && nce > 2) {
    std::vector<int64_t> cx(nce + 1, 0), cadj, vw(nce);
    std::vector<int> mark(nc, -1);
    cadj.reserve((size_t)xadj[n]);
    for (int v = 0; v < nce; ++v) {
      mark[v] = v;
      int mem[2] = {cfirst[v], csecond[v]};
      for (int m = 0; m < 2; ++m) {
        if (mem[m] < 0) continue;
        for (int64_t p = xadj[mem[m]]; p < xadj[mem[m] + 1]; ++p) {
          int w = cnode[adj[p]];
          if (w < nce && mark[w] != v) { mark[w] = v; cadj.push_back(w); }
        }
      }
      cx[v + 1] = (int64_t)cadj.size();
      vw[v] = csecond[v] >= 0 ? 2 : 1;
    }
    if (!cadj.empty()) {
      int64_t nv = nce;
      std::vector<int64_t> mp(nce), mip(nce);
      int64_t mopt[40];
      METIS_SetDefaultOptions(mopt);
      int rc = METIS_NodeND(&nv, cx.data(), cadj.data(), vw.data(), mopt, mp.data(), mip.data());
      if (rc != 1) { err = "METIS_NodeND failed"; return -3; }
      for (int v = 0; v < nce; ++v) cperm[v] = (int)mp[v];  // new position v holds compressed node mp[v]
    }
  }
  S.t_order = now_s() - t_ord0;

  std::vector<int> perm(n), iperm(n);
  {
    int q = 0;
    for (int v = 0; v < nc; ++v) {
      int cn = cperm[v];
      perm[q++] = cfirst[cn];
      if (csecond[cn] >= 0) perm[q++] = csecond[cn];
    }
    for (int k = 0; k < n; ++k) iperm[perm[k]] = k;
    // Saddle rows without a partner.  For every prefix of the elimination order the eliminated saddle rows
    // must be matchable into the eliminated primal columns (Hall's condition), otherwise a pivot is
    // structurally zero.  A partnered row satisfies it by construction (its primal sits right before it).  For an
    // unpartnered row s0 we look for an augmenting path (of any length) in a SHADOW copy of the matching and
    // eliminate s0 only after every primal column on that path - without changing the real pairs.
    bool moved = false;
    std::vector<double> key(n);
    for (int k = 0; k < n; ++k) key[perm[k]] = (double)k;
    {
      std::vector<int> shadow(partner);
      std::vector<int> visit(n, -1), from_s(n, -1), queue;
      for (int s0 = 0; s0 < n; ++s0) {
        if (!saddle[s0] || partner[s0] >= 0 || is_sc[s0]) continue;
        queue.clear();
        queue.push_back(s0);
        int found_x = -1;
        for (size_t qh = 0; qh < queue.size() && found_x < 0; ++qh) {
          int sq = queue[qh];
          for (int64_t p = xadj[sq]; p < xadj[sq + 1]; ++p) {
            int x = adj[p];
            if (saddle[x] || is_sc[x] || visit[x] == s0 || !(adjw[p] > 0.0)) continue;
            visit[x] = s0;
            from_s[x] = sq;
            if (shadow[x] < 0) { found_x = x; break; }
            queue.push_back(shadow[x]);
          }
        }
        int last = -1;
        if (found_x >= 0) {
          int x = found_x;
          while (true) {
            last = std::max(last, iperm[x]);
            int sq = from_s[x];
            int prev_x = shadow[sq];
            shadow[sq] = x; shadow[x] = sq;
            if (sq == s0) break;
            x = prev_x;
          }
        }
        for (int64_t p = xadj[s0]; p < xadj[s0 + 1]; ++p) last = std::max(last, iperm[adj[p]]);
        last = std::min(last, n - m - 1);   // never into the Schur block
        if (last > iperm[s0]) {
          // do not split the pair (primal at `last`, its saddle partner at last+1)
          const int xl = perm[last];
          if (partner[xl] >= 0 && iperm[partner[xl]] == last + 1) last += 1;
          key[s0] = (double)last + 0.5;
          moved = true;
        }
      }
    }
    if (moved) {
      std::stable_sort(perm.begin(), perm.end(), [&](int a, int b2) { return key[a] < key[b2]; });
      for (int k = 0; k < n; ++k) iperm[perm[k]] = k;
    }
  }

  // ---- 5. etree, postorder, relabel -----------------------------------------------------------
  // The elimination tree, the column counts and the row structures see the path sc[0]-sc[1]-...-sc[m-1] as extra edges:
  // S is then a chain at the top of the tree, which the postorder (roots ascending) keeps last and in order.  The
  // numeric pattern (step 9) does not see them.
  std::vector<int64_t> xadj_p;
  std::vector<int> adj_p;
  if (m > 1) {
    std::vector<int> nxt(n, -1), prv(n, -1);
    for (int i = 0; i + 1 < m; ++i) { nxt[sc[i]] = sc[i + 1]; prv[sc[i + 1]] = sc[i]; }
    xadj_p.assign(n + 1, 0);
    for (int i = 0; i < n; ++i) xadj_p[i + 1] = xadj_p[i] + (xadj[i + 1] - xadj[i]) + (nxt[i] >= 0) + (prv[i] >= 0);
    adj_p.resize((size_t)xadj_p[n]);
    for (int i = 0; i < n; ++i) {
      int64_t q = xadj_p[i];
      for (int64_t p = xadj[i]; p < xadj[i + 1]; ++p) adj_p[q++] = adj[p];
      if (nxt[i] >= 0) adj_p[q++] = nxt[i];
      if (prv[i] >= 0) adj_p[q++] = prv[i];
    }
  }
  const std::vector<int64_t>& gx = m > 1 ? xadj_p : xadj;
  const std::vector<int>& ga = m > 1 ? adj_p : adj;
  std::vector<int> parent;
  etree_from_graph(n, gx, ga, perm, iperm, parent);
  {
    std::vector<int> post;
    postorder(n, parent, post);
    std::vector<int> perm2(n);
    for (int t = 0; t < n; ++t) perm2[t] = perm[post[t]];
    perm.swap(perm2);
    for (int k = 0; k < n; ++k) iperm[perm[k]] = k;
    etree_from_graph(n, gx, ga, perm, iperm, parent);
  }

  // children lists (ascending)
  std::vector<int> chead(n, -1), cnext(n, -1);
  for (int j = n - 1; j >= 0; --j) if (parent[j] >= 0) { cnext[j] = chead[parent[j]]; chead[parent[j]] = j; }

  // ---- 6. column counts (pass 1) --------------------------------------------------------------
  // Skeleton-graph algorithm (Gilbert, Ng, Peyton 1994): entry (i, j), i > j, of the permuted matrix makes j a LEAF of the
  // row subtree of i iff j's first descendant lies beyond every leaf seen so far; every new leaf adds one to the count of j
  // and takes one from the least common ancestor with the previous leaf (found with a path-halving disjoint-set forest).
  // O(nnz(A) alpha(n)) instead of walking the nnz(L) structure.  The columns are already numbered in postorder, so the
  // first descendant of j is j - size(j) + 1.
  std::vector<int> cc(n, 1);
  {
    std::vector<int> first(n), delta(n), maxfirst(n, -1), prevleaf(n, -1), anc(n);
    {
      std::vector<int> sz(n, 1);
      for (int j = 0; j < n; ++j) if (parent[j] >= 0) sz[parent[j]] += sz[j];
      for (int j = 0; j < n; ++j) { first[j] = j - sz[j] + 1; delta[j] = (sz[j] == 1) ? 1 : 0; }
    }
    std::iota(anc.begin(), anc.end(), 0);
    auto find = [&](int v) {
      while (anc[v] != v) { anc[v] = anc[anc[v]]; v = anc[v]; }
      return v;
    };
    for (int j = 0; j < n; ++j) {
      if (parent[j] >= 0) delta[parent[j]]--;        // j is not a root: its parent's count loses the overlap
      const int old = perm[j];
      for (int64_t p = gx[old]; p < gx[old + 1]; ++p) {
        const int i = iperm[ga[p]];
        if (i <= j || first[j] <= maxfirst[i]) continue;
        maxfirst[i] = first[j];
        const int jprev = prevleaf[i];
        prevleaf[i] = j;
        delta[j]++;                                   // j is a leaf of the row subtree of i
        if (jprev >= 0) delta[find(jprev)]--;         // ... a subsequent one: the path above the lca was counted before
      }
      if (parent[j] >= 0) anc[j] = parent[j];
    }
    for (int j = 0; j < n; ++j) cc[j] = delta[j];
    for (int j = 0; j < n; ++j) if (parent[j] >= 0) cc[parent[j]] += cc[j];
    if (getenv("B200_SYMBOLIC_CHECK")) {              // debug: the explicit column structures, one column at a time
      std::vector<std::vector<int>> st(n);
      std::vector<int> mark(n, -1);
      long long bad = 0;
      for (int j = 0; j < n; ++j) {
        std::vector<int>& out = st[j];
        int old2 = perm[j];
        for (int64_t p = gx[old2]; p < gx[old2 + 1]; ++p) {
          int i = iperm[ga[p]];
          if (i > j && mark[i] != j) { mark[i] = j; out.push_back(i); }
        }
        for (int c = chead[j]; c >= 0; c = cnext[c]) {
          for (int i : st[c]) if (i != j && mark[i] != j) { mark[i] = j; out.push_back(i); }
          std::vector<int>().swap(st[c]);
        }
        if (cc[j] != (int)out.size() + 1) ++bad;
      }
      fprintf(stderr, "[symbolic] column-count check: %lld of %d columns differ\n", bad, n);
      if (bad) { err = "column count self-check failed"; return -6; }
    }
    for (int j = 0; j < n; ++j) S.nnzL_true += cc[j];
  }

  // ---- 7. supernode partition -----------------------------------------------------------------
  std::vector<char> link(n, 0);  // link[j]: j and j+1 share a supernode
  // the Schur block is one supernode of its own, whatever the merges below would do
  auto sc_links = [&]() {
    if (m == 0) return;
    link[n - m - 1] = 0;
    for (int j = n - m; j + 1 < n; ++j) link[j] = 1;
  };
  if (n <= opt.dense_n) {
    for (int j = 0; j + 1 < n; ++j) link[j] = 1;
    sc_links();
  } else {
    std::vector<int> sz(n, 1);
    for (int j = 0; j < n; ++j) if (parent[j] >= 0) sz[parent[j]] += sz[j];
    for (int v = 0; v < n; ++v) {
      if (sz[v] <= opt.leaf_k && sz[v] > 1 && (parent[v] < 0 || sz[parent[v]] > opt.leaf_k))
        for (int j = v - sz[v] + 1; j < v; ++j) link[j] = 1;
    }
    for (int j = 1; j < n; ++j)
      if (parent[j - 1] == j && cc[j - 1] == cc[j] + 1) link[j - 1] = 1;
    // saddle pairs must share a supernode (primal at p, saddle row at p+1)
    for (int i = 0; i < n; ++i) if (saddle[i] && partner[i] >= 0) {
      int pc = iperm[i], px = iperm[partner[i]];
      if (pc == px + 1 && parent[px] == pc) link[px] = 1;
    }
    sc_links();
    // relaxed amalgamation of a contiguous last child into its parent, cumulative criterion
    int gstart = 0;
    int64_t gtrue = 0;
    int b = 0;
    while (b < n) {
      // current fundamental piece [b, e]
      int e = b;
      while (e + 1 < n && link[e]) ++e;
      int64_t ptrue = 0;
      for (int j = b; j <= e; ++j) ptrue += cc[j];
      gtrue += ptrue;
      // boundary after e
      if (e + 1 < n - m && parent[e] == e + 1) {
        int e2 = e + 1;
        while (e2 + 1 < n && link[e2]) ++e2;
        int64_t ntrue = 0;
        for (int j = e + 1; j <= e2; ++j) ntrue += cc[j];
        int64_t K = e2 - gstart + 1, rp = cc[e2] - 1;
        int64_t store = K * (K + 1) / 2 + K * rp;
        if (K <= opt.relax_small || (double)store <= (1.0 + opt.relax_frac) * (double)(gtrue + ntrue)) {
          link[e] = 1;
        } else { gstart = e + 1; gtrue = 0; }
      } else { gstart = e + 1; gtrue = 0; }
      b = e + 1;
    }
  }
  std::vector<int> sn_of(n);
  S.sn_start.clear();
  for (int j = 0; j < n; ++j) {
    if (j == 0 || !link[j - 1]) S.sn_start.push_back(j);
    sn_of[j] = (int)S.sn_start.size() - 1;
  }
  S.nsn = (int)S.sn_start.size();
  S.sn_start.push_back(n);
  const int nsn = S.nsn;
  S.sn_parent.assign(nsn, -1);
  for (int s = 0; s < nsn; ++s) {
    int last = S.sn_start[s + 1] - 1;
    S.sn_parent[s] = parent[last] >= 0 ? sn_of[parent[last]] : -1;
  }
  S.child_ptr.assign(nsn + 1, 0);
  for (int s = 0; s < nsn; ++s) if (S.sn_parent[s] >= 0) S.child_ptr[S.sn_parent[s] + 1]++;
  for (int s = 0; s < nsn; ++s) S.child_ptr[s + 1] += S.child_ptr[s];
  S.child_idx.resize(S.child_ptr[nsn]);
  {
    std::vector<int> pos(S.child_ptr.begin(), S.child_ptr.end() - 1);
    for (int s = 0; s < nsn; ++s) if (S.sn_parent[s] >= 0) S.child_idx[pos[S.sn_parent[s]]++] = s;
  }

  // ---- 8. supernodal row structures (pass 2) --------------------------------------------------
  S.rows_ptr.assign(nsn + 1, 0);
  {
    std::vector<int> mark(n, -1);
    std::vector<int> buf;
    for (int s = 0; s < nsn; ++s) {
      int a = S.sn_start[s], e = S.sn_start[s + 1];
      buf.clear();
      for (int j = a; j < e; ++j) {
        int old = perm[j];
        for (int64_t p = gx[old]; p < gx[old + 1]; ++p) {
          int i = iperm[ga[p]];
          if (i >= e && mark[i] != s) { mark[i] = s; buf.push_back(i); }
        }
      }
      for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
        int c = S.child_idx[q];
        for (int64_t p = S.rows_ptr[c]; p < S.rows_ptr[c + 1]; ++p) {
          int i = S.rows[p];
          if (i >= e && mark[i] != s) { mark[i] = s; buf.push_back(i); }
        }
      }
      std::sort(buf.begin(), buf.end());
      S.rows.insert(S.rows.end(), buf.begin(), buf.end());
      S.rows_ptr[s + 1] = (int64_t)S.rows.size();
    }
  }
  // relative indices into the parent front
  S.rel.assign(S.rows.size(), -1);
  for (int s = 0; s < nsn; ++s) {
    int p = S.sn_parent[s];
    if (p < 0) {
      if (S.rows_ptr[s + 1] != S.rows_ptr[s]) { err = "internal: root supernode with rows"; return -4; }
      continue;
    }
    int pa = S.sn_start[p], pe = S.sn_start[p + 1], kp = pe - pa;
    int64_t q = S.rows_ptr[p];
    for (int64_t t = S.rows_ptr[s]; t < S.rows_ptr[s + 1]; ++t) {
      int i = S.rows[t];
      if (i < pe) {
        if (i < pa) { err = "internal: child row below parent start"; return -4; }
        S.rel[t] = i - pa;
      } else {
        while (q < S.rows_ptr[p + 1] && S.rows[q] < i) ++q;
        if (q >= S.rows_ptr[p + 1] || S.rows[q] != i) { err = "internal: child row missing in parent"; return -4; }
        S.rel[t] = kp + (int)(q - S.rows_ptr[p]);
      }
    }
  }

  // ---- 9. unique entries in final order, assembly maps ----------------------------------------
  {
    std::vector<Ent> k2((size_t)nu);
    for (int64_t u = 0; u < nu; ++u) {
      int a = iperm[ur[u]], b2 = iperm[uc[u]];
      k2[u] = Ent{std::min(a, b2), std::max(a, b2), (int)u};
    }
    sort_entries(n, k2);
    std::vector<int> rank((size_t)nu);
    S.u_row.resize(nu); S.u_col.resize(nu); S.u_dst.resize(nu); S.u_dst64.resize(nu);
    S.uent_ptr.assign(nsn + 1, 0);
    for (int64_t q = 0; q < nu; ++q) {
      int u = k2[q].id;
      rank[u] = (int)q;
      int c = k2[q].c, r = k2[q].r;
      int s = sn_of[c];
      int a = S.sn_start[s], e = S.sn_start[s + 1], k = e - a;
      int fr = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
      int lrow;
      if (r < e) lrow = r - a;
      else {
        const int* rb = S.rows.data() + S.rows_ptr[s];
        const int* re = S.rows.data() + S.rows_ptr[s + 1];
        const int* it = std::lower_bound(rb, re, r);
        if (it == re || *it != r) { err = "internal: entry row missing in front"; return -4; }
        lrow = k + (int)(it - rb);
      }
      int lcol = c - a;
      S.u_row[q] = ur[u]; S.u_col[q] = uc[u];
      S.u_dst64[q] = (int64_t)lrow + (int64_t)lcol * fr;
      S.u_dst[q] = ((uint32_t)lcol << 16) | (uint32_t)(lrow & 0xffff);
      S.uent_ptr[s + 1]++;
    }
    for (int s = 0; s < nsn; ++s) S.uent_ptr[s + 1] += S.uent_ptr[s];
    S.t2u.resize(nnz);
    for (int64_t e = 0; e < nnz; ++e) S.t2u[e] = rank[t2u0[e]];
    S.useg_ptr.assign(nu + 1, 0);
    for (int64_t e = 0; e < nnz; ++e) S.useg_ptr[S.t2u[e] + 1]++;
    for (int64_t u = 0; u < nu; ++u) S.useg_ptr[u + 1] += S.useg_ptr[u];
    S.useg_src.resize(nnz);
    std::vector<int64_t> pos(S.useg_ptr.begin(), S.useg_ptr.end() - 1);
    for (int64_t e = 0; e < nnz; ++e) S.useg_src[pos[S.t2u[e]]++] = (int)e;
  }

  // ---- 10. offsets, levels, statistics ---------------------------------------------------------
  S.L_off.assign(nsn + 1, 0);
  S.cb_off.assign(nsn + 1, 0);
  S.sn_level.assign(nsn, 0);
  for (int s = 0; s < nsn; ++s) {
    int64_t k = S.k(s), r = S.r(s), f = k + r;
    // keep every panel 16-byte aligned (even element offsets) for vector loads
    int64_t lsz = f * k; lsz += lsz & 1;
    int64_t csz = r * r; csz += csz & 1;
    S.L_off[s + 1] = S.L_off[s] + lsz;
    S.cb_off[s + 1] = S.cb_off[s] + csz;
    S.nnzL += k * (k + 1) / 2 + k * r;
    S.flops_panel += (double)k * k * k / 3.0 + (double)k * k * r;
    S.flops_schur += (double)k * r * (r + 1);
    S.cb_total += r * r;
    S.max_front = std::max<int>(S.max_front, (int)f);
    S.max_k = std::max<int>(S.max_k, (int)k);
    if (f >= 65536) { err = "front too large (>= 65536)"; return -5; }
  }
  for (int s = 0; s < nsn; ++s) {
    int p = S.sn_parent[s];
    if (p >= 0) S.sn_level[p] = std::max(S.sn_level[p], S.sn_level[s] + 1);
  }
  S.nlevels = 0;
  for (int s = 0; s < nsn; ++s) S.nlevels = std::max(S.nlevels, S.sn_level[s] + 1);
  S.level_sn.resize(nsn);
  std::iota(S.level_sn.begin(), S.level_sn.end(), 0);
  std::stable_sort(S.level_sn.begin(), S.level_sn.end(), [&](int a, int b2) {
    if (S.sn_level[a] != S.sn_level[b2]) return S.sn_level[a] < S.sn_level[b2];
    return S.f(a) > S.f(b2);
  });
  S.level_ptr.assign(S.nlevels + 1, 0);
  for (int s = 0; s < nsn; ++s) S.level_ptr[S.sn_level[s] + 1]++;
  for (int l = 0; l < S.nlevels; ++l) S.level_ptr[l + 1] += S.level_ptr[l];

  S.perm = perm;
  S.iperm = iperm;
  S.t_symbolic = now_s() - t0 - S.t_order;
  return 0;
}


int shard_plan(const Symbolic& S, int world, std::vector<int>& owner) {
  const int nsn = S.nsn;
  owner.assign(nsn, 0);
  if (world <= 1 || nsn == 0) return 1;
  std::vector<double> w(nsn), sub(nsn);
  for (int s = 0; s < nsn; ++s) {
    const double k = S.k(s), r = S.r(s);
    w[s] = k * k * k / 3.0 + k * k * r + k * r * (r + 1.0) + 50.0 * (k + r);  // + a latency term per front
    sub[s] = w[s];
  }
  for (int s = 0; s < nsn; ++s) if (S.sn_parent[s] >= 0) sub[S.sn_parent[s]] += sub[s];  // children precede parents
  std::vector<char> top(nsn, 0);
  std::vector<int> frontier;
  for (int s = 0; s < nsn; ++s) if (S.sn_parent[s] < 0) frontier.push_back(s);
  double below = 0;
  for (int s : frontier) below += sub[s];
  // expand the heaviest subtree until the cut exposes enough balanced subtrees
  for (int iter = 0; iter < nsn; ++iter) {
    int bi = -1;
    for (int q = 0; q < (int)frontier.size(); ++q)
      if (S.child_ptr[frontier[q] + 1] > S.child_ptr[frontier[q]] && (bi < 0 || sub[frontier[q]] > sub[frontier[bi]])) bi = q;
    if (bi < 0) break;
    const bool enough = (int)frontier.size() >= 4 * world && sub[frontier[bi]] <= below / (2.0 * world);
    if (enough) break;
    const int s = frontier[bi];
    top[s] = 1;
    below -= w[s];
    frontier[bi] = frontier.back();
    frontier.pop_back();
    for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) frontier.push_back(S.child_idx[q]);
  }
  // LPT assignment of the subtrees
  std::sort(frontier.begin(), frontier.end(), [&](int a, int b) { return sub[a] != sub[b] ? sub[a] > sub[b] : a < b; });
  std::vector<double> load(world, 0.0);
  std::vector<int> root_owner(nsn, -1);
  for (int s : frontier) {
    int g = 0;
    for (int q = 1; q < world; ++q) if (load[q] < load[g]) g = q;
    load[g] += sub[s];
    root_owner[s] = g;
  }
  // propagate down (parents have larger indices than children)
  for (int s = nsn - 1; s >= 0; --s) {
    if (top[s]) owner[s] = -1;
    else if (root_owner[s] >= 0) owner[s] = root_owner[s];
    else owner[s] = owner[S.sn_parent[s]];
  }
  return (int)frontier.size();
}

}  // namespace b200
