// TEST / BENCH INFRASTRUCTURE: runs the reference's UNMODIFIED interior-point loop (libipopt built from
// the reference sources into oracle/_ref) on the reference's own benchmark TNLPs (oracle/_ref/lib/libreftnlp.so:
// examples/ScalableProblems/*.cpp, examples/hs071_cpp/hs071_nlp.cpp) with the KKT linear solver injected
// through the reference's custom-solver hook, exactly as SURVEY.md section 8(b) describes:
//   new AlgorithmBuilder(new StdAugSystemSolver(*new TSymLinearSolver(iface, NULL)), name) + linear_solver=custom
//   (reference src/Algorithm/IpAlgBuilder.hpp:55-58, IpAlgBuilder.cpp:576-584; driver modelled on
//    examples/ScalableProblems/solve_problem.cpp:103-260).
// Backends: "b200" = the product (libb200ldlt.so via ipopt_b200/plugin), "oracle" = oracle/cpu_ldlt.cpp.
#include <dlfcn.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "B200LdltSolverInterface.hpp"
#include "IpAlgBuilder.hpp"
#include "IpIpoptApplication.hpp"
#include "IpSolveStatistics.hpp"
#include "IpStdAugSystemSolver.hpp"
#include "IpTNLPAdapter.hpp"
#include "IpTSymLinearSolver.hpp"
#include "RegisteredTNLP.hpp"
#include "hs071_nlp.hpp"

#include "LuksanVlcek1.hpp"
REGISTER_TNLP(LuksanVlcek1(0, 0), LukVlE1)
REGISTER_TNLP(LuksanVlcek1(-1., 0.), LukVlI1)
#include "LuksanVlcek2.hpp"
REGISTER_TNLP(LuksanVlcek2(0, 0), LukVlE2)
#include "LuksanVlcek3.hpp"
REGISTER_TNLP(LuksanVlcek3(0, 0), LukVlE3)
#include "LuksanVlcek4.hpp"
REGISTER_TNLP(LuksanVlcek4(0, 0), LukVlE4)
#include "LuksanVlcek5.hpp"
REGISTER_TNLP(LuksanVlcek5(0, 0), LukVlE5)
#include "MittelmannBndryCntrlDiri.hpp"
REGISTER_TNLP(MittelmannBndryCntrlDiri1, MBndryCntrl1)
REGISTER_TNLP(MittelmannBndryCntrlDiri2, MBndryCntrl2)
REGISTER_TNLP(MittelmannBndryCntrlDiri3, MBndryCntrl3)
REGISTER_TNLP(MittelmannBndryCntrlDiri4, MBndryCntrl4)
#include "MittelmannBndryCntrlNeum.hpp"
REGISTER_TNLP(MittelmannBndryCntrlNeum1, MBndryCntrl5)
#include "MittelmannDistCntrlDiri.hpp"
REGISTER_TNLP(MittelmannDistCntrlDiri1, MDistCntrl1)
REGISTER_TNLP(MittelmannDistCntrlDiri2, MDistCntrl2)
REGISTER_TNLP(MittelmannDistCntrlDiri3, MDistCntrl3)
REGISTER_TNLP(MittelmannDistCntrlDiri3a, MDistCntrl3a)
#include "MittelmannDistCntrlNeumA.hpp"
REGISTER_TNLP(MittelmannDistCntrlNeumA1, MDistCntrl4)

using namespace Ipopt;

// ---- oracle backend glue (C ABI of oracle/cpu_ldlt.cpp) ---------------------------------------------------
extern "C" {
void* oracle_ldlt_create(double, double, int, int);
void oracle_ldlt_destroy(void*);
int oracle_ldlt_analyse(void*, int, int, const int*, const int*);
double* oracle_ldlt_values_ptr(void*);
int oracle_ldlt_factor(void*, int, int, int*);
int oracle_ldlt_solve(void*, int, double*);
int oracle_ldlt_num_neg(void*);
int oracle_ldlt_increase_quality(void*);
}
static void* orc_create(double pivtol, double pivtolmax, int scaling, int verbose, int)
{
   // comparator defaults follow the reference's MUMPS adapter: pivtol 1e-6, pivtolmax 0.1
   // (IpMumpsSolverInterface.cpp:137-158); the b200_* options are not applied to the oracle.
   (void) pivtol; (void) pivtolmax; (void) scaling;
   // control experiments (tests/test_dual_spread_control.py): the same oracle with another pivot threshold / scaling
   // (and ORACLE_METIS_SEED, read by oracle/cpu_ldlt.cpp) to measure the solver-to-solver spread of the final iterates
   const char* ep = getenv("ORACLE_PIVTOL");
   const char* es = getenv("ORACLE_SCALING");
   return oracle_ldlt_create(ep ? atof(ep) : 1e-6, 0.1, es ? atoi(es) : 1, verbose);
}
static const LdltBackend oracle_backend = {"cpu-oracle-ldlt", orc_create, oracle_ldlt_destroy, oracle_ldlt_analyse,
                                           oracle_ldlt_values_ptr, oracle_ldlt_factor, oracle_ldlt_solve,
                                           oracle_ldlt_num_neg, oracle_ldlt_increase_quality, NULL, NULL};

// ---- TNLP wrapper that records the final iterate -----------------------------------------------------------
class CapturingTNLP: public TNLP
{
public:
   CapturingTNLP(SmartPtr<TNLP> t) : t_(t), obj(0), status(-1) { }
   bool get_nlp_info(Index& n, Index& m, Index& nj, Index& nh, IndexStyleEnum& is) { return t_->get_nlp_info(n, m, nj, nh, is); }
   bool get_bounds_info(Index n, Number* xl, Number* xu, Index m, Number* gl, Number* gu) { return t_->get_bounds_info(n, xl, xu, m, gl, gu); }
   bool get_scaling_parameters(Number& os, bool& ux, Index n, Number* xs, bool& ug, Index m, Number* gs) { return t_->get_scaling_parameters(os, ux, n, xs, ug, m, gs); }
   bool get_starting_point(Index n, bool ix, Number* x, bool iz, Number* zl, Number* zu, Index m, bool il, Number* l) { return t_->get_starting_point(n, ix, x, iz, zl, zu, m, il, l); }
   bool eval_f(Index n, const Number* x, bool nx, Number& o) { return t_->eval_f(n, x, nx, o); }
   bool eval_grad_f(Index n, const Number* x, bool nx, Number* g) { return t_->eval_grad_f(n, x, nx, g); }
   bool eval_g(Index n, const Number* x, bool nx, Index m, Number* g) { return t_->eval_g(n, x, nx, m, g); }
   bool eval_jac_g(Index n, const Number* x, bool nx, Index m, Index ne, Index* ir, Index* jc, Number* v) { return t_->eval_jac_g(n, x, nx, m, ne, ir, jc, v); }
   bool eval_h(Index n, const Number* x, bool nx, Number of, Index m, const Number* l, bool nl, Index ne, Index* ir, Index* jc, Number* v) { return t_->eval_h(n, x, nx, of, m, l, nl, ne, ir, jc, v); }
   void finalize_solution(SolverReturn st, Index n, const Number* x, const Number* zl, const Number* zu, Index m,
                          const Number* g, const Number* l, Number o, const IpoptData* d, IpoptCalculatedQuantities* q)
   {
      xs.assign(x, x + n); zls.assign(zl, zl + n); zus.assign(zu, zu + n); ls.assign(l, l + m); obj = o; status = (int) st;
      t_->finalize_solution(st, n, x, zl, zu, m, g, l, o, d, q);
   }
   SmartPtr<TNLP> t_;
   std::vector<Number> xs, zls, zus, ls;
   Number obj;
   int status;
};

static double wall_now()
{
   using namespace std::chrono;
   return duration<double>(steady_clock::now().time_since_epoch()).count();
}

extern "C" int omp_get_max_threads(void);

int main(int argc, char** argv)
{
   // The host BLAS (OpenBLAS, pthread build) sizes its pool from the machine's hardware threads, not from the
   // container's quota; on a many-core GPU box that turns every level-1 BLAS call of the IP loop into a storm of
   // spinning workers.  Level-1 ops on <1e6 doubles are memory-bound anyway: keep the host BLAS single-threaded
   // unless asked otherwise.
   // (looked up at run time: the BLAS is libipopt.so's dependency, not linked here; absent for a non-OpenBLAS BLAS)
   {
      const char* e = getenv("B200_HOST_BLAS_THREADS");
      void (*set_threads)(int) = (void (*)(int))dlsym(RTLD_DEFAULT, "openblas_set_num_threads");
      if( set_threads ) set_threads(e ? atoi(e) : 1);
   }
   std::string backend = "b200", problem = "hs071", json_path, final_path, dump_prefix;
   bool reopt = false;   // second solve of the same NLP with warm_start_same_structure=yes (ReOptimizeNLP)
   int N = 0, print_level = 5;
   std::vector<std::pair<std::string, std::string> > opts;
   std::vector<int> dump_which;
   for( int a = 1; a < argc; ++a )
   {
      std::string s = argv[a];
      if( s == "--backend" && a + 1 < argc ) backend = argv[++a];
      else if( s == "--problem" && a + 1 < argc ) problem = argv[++a];
      else if( s == "--N" && a + 1 < argc ) N = atoi(argv[++a]);
      else if( s == "--json" && a + 1 < argc ) json_path = argv[++a];
      else if( s == "--final" && a + 1 < argc ) final_path = argv[++a];
      else if( s == "--print-level" && a + 1 < argc ) print_level = atoi(argv[++a]);
      else if( s == "--dump" && a + 1 < argc ) dump_prefix = argv[++a];
      else if( s == "--reopt" ) reopt = true;
      else if( s == "--dump-iters" && a + 1 < argc )
      {
         char* p = argv[++a];
         while( *p ) { dump_which.push_back((int) strtol(p, &p, 10)); if( *p == ',' ) ++p; }
      }
      else if( s == "--opt" && a + 1 < argc )
      {
         std::string kv = argv[++a];
         size_t eq = kv.find('=');
         if( eq == std::string::npos ) { fprintf(stderr, "bad --opt %s\n", kv.c_str()); return 2; }
         opts.push_back(std::make_pair(kv.substr(0, eq), kv.substr(eq + 1)));
      }
      else { fprintf(stderr, "unknown argument %s\n", s.c_str()); return 2; }
   }

   SmartPtr<TNLP> inner;
   if( problem == "hs071" ) inner = new HS071_NLP();
   else
   {
      SmartPtr<RegisteredTNLP> r = RegisteredTNLPs::GetTNLP(problem);
      if( !IsValid(r) ) { fprintf(stderr, "unknown problem %s\n", problem.c_str()); return 2; }
      if( N <= 0 || !r->InitializeProblem(N) ) { fprintf(stderr, "bad N\n"); return 2; }
      inner = GetRawPtr(r);
   }
   SmartPtr<CapturingTNLP> tnlp = new CapturingTNLP(inner);

   // "ma97": NO custom hook at all -- the stock reference code path  linear_solver=ma97 + hsllib=<libb200ldlt.so>  (the
   // reference dlopen()s the library and binds the seven ma97_*_d symbols of ipopt_b200/csrc/hsl_shim.cpp)
   const bool via_hsllib = backend == "ma97";
   const LdltBackend* be = backend == "oracle" ? &oracle_backend : GetB200LdltBackend();
   SmartPtr<B200LdltSolverInterface> iface = new B200LdltSolverInterface(be);
   if( !dump_prefix.empty() ) iface->SetDump(dump_prefix, dump_which);

   SmartPtr<IpoptApplication> app = IpoptApplicationFactory();
   B200LdltSolverInterface::RegisterOptions(app->RegOptions());
   if( via_hsllib )
   {
      const char* lib = getenv("B200_HSLLIB");
      if( !lib ) { fprintf(stderr, "--backend ma97 needs B200_HSLLIB=<path to libb200ldlt.so>\n"); return 2; }
      app->Options()->SetStringValue("linear_solver", "ma97");
      app->Options()->SetStringValue("hsllib", lib);
   }
   else
      app->Options()->SetStringValue("linear_solver", "custom");
   app->Options()->SetIntegerValue("print_level", print_level);
   if( problem == "hs071" )
   {  // the settings of reference examples/hs071_cpp/hs071_main.cpp:33-35
      app->Options()->SetNumericValue("tol", 3.82e-6);
      app->Options()->SetStringValue("mu_strategy", "adaptive");
   }
   for( size_t q = 0; q < opts.size(); ++q )
   {
      const std::string& k = opts[q].first;
      const std::string& v = opts[q].second;
      char* end = NULL;
      long iv = strtol(v.c_str(), &end, 10);
      bool ok;
      if( *end == 0 && !v.empty() ) { ok = app->Options()->SetIntegerValue(k, (Index) iv); if( !ok ) ok = app->Options()->SetNumericValue(k, (Number) iv); }
      else
      {
         double dv = strtod(v.c_str(), &end);
         if( *end == 0 && !v.empty() ) ok = app->Options()->SetNumericValue(k, dv);
         else ok = app->Options()->SetStringValue(k, v);
      }
      if( !ok ) { fprintf(stderr, "could not set option %s=%s\n", k.c_str(), v.c_str()); return 2; }
   }
   ApplicationReturnStatus st = app->Initialize();
   if( st != Solve_Succeeded ) { fprintf(stderr, "Initialize failed\n"); return 3; }

   SmartPtr<SymLinearSolver> sls = new TSymLinearSolver(GetRawPtr(iface), NULL);
   SmartPtr<AugSystemSolver> aug = new StdAugSystemSolver(*sls);
   SmartPtr<AlgorithmBuilder> builder = new AlgorithmBuilder(aug, be->name);
   SmartPtr<NLP> nlp = new TNLPAdapter(GetRawPtr(tnlp), app->Jnlst());

   double t0 = wall_now();
   if( via_hsllib ) st = app->OptimizeTNLP(GetRawPtr(tnlp));
   else st = app->OptimizeNLP(nlp, builder);
   double total = wall_now() - t0;
   int reopt_status = -99, reopt_iters = -1, n_factor_first = iface->GetStats().n_factor;
   if( reopt && !via_hsllib )
   {
      // the reference's warm-start contract (IpMumpsSolverInterface.cpp:227-236): same structure => the adapter keeps its
      // handle and symbolic analysis, InitializeStructure is answered without re-analysing
      app->Options()->SetStringValue("warm_start_same_structure", "yes");
      ApplicationReturnStatus st2 = app->ReOptimizeNLP(nlp);
      reopt_status = (int) st2;
      if( IsValid(app->Statistics()) ) reopt_iters = app->Statistics()->IterationCount();
   }

   int iters = -1;
   double obj = 0;
   if( IsValid(app->Statistics()) ) { iters = app->Statistics()->IterationCount(); obj = app->Statistics()->FinalObjective(); }
   const B200LdltSolverInterface::Stats& S = iface->GetStats();
   char buf[2048];
   snprintf(buf, sizeof(buf),
            "{\"backend\": \"%s\", \"problem\": \"%s\", \"N\": %d, \"status\": %d, \"iterations\": %d, \"objective\": %.17g, "
            "\"kkt_dim\": %d, \"kkt_nnz\": %d, \"n_factor\": %d, \"n_solve\": %d, \"n_rhs\": %d, \"n_singular\": %d, "
            "\"n_wrong_inertia\": %d, \"t_first_factor_s\": %.6f, \"t_factor_s\": %.6f, \"t_solve_s\": %.6f, \"t_total_s\": %.6f, \"host_threads\": %d, "
            "\"n_analyse\": %d, \"reopt_status\": %d, \"reopt_iterations\": %d, \"n_factor_first\": %d}",
            via_hsllib ? "ma97-shim(b200-ldlt)" : be->name, problem.c_str(), N, (int) st, iters, obj, S.dim, S.nonzeros, S.n_factor, S.n_solve, S.n_rhs,
            S.n_singular, S.n_wrong_inertia, S.t_first_factor, S.t_factor, S.t_solve, total, omp_get_max_threads(),
            S.n_analyse, reopt_status, reopt_iters, n_factor_first);
   printf("DRIVER_JSON %s\n", buf);
   if( !json_path.empty() ) { FILE* fp = fopen(json_path.c_str(), "w"); if( fp ) { fprintf(fp, "%s\n", buf); fclose(fp); } }
   if( !final_path.empty() )
   {  // int32 n, m; f64 obj; f64 x[n], z_L[n], z_U[n], lambda[m]
      FILE* fp = fopen(final_path.c_str(), "wb");
      if( fp )
      {
         int hdr[2] = {(int) tnlp->xs.size(), (int) tnlp->ls.size()};
         fwrite(hdr, sizeof(int), 2, fp);
         fwrite(&tnlp->obj, sizeof(double), 1, fp);
         if( hdr[0] ) { fwrite(&tnlp->xs[0], 8, hdr[0], fp); fwrite(&tnlp->zls[0], 8, hdr[0], fp); fwrite(&tnlp->zus[0], 8, hdr[0], fp); }
         if( hdr[1] ) fwrite(&tnlp->ls[0], 8, hdr[1], fp);
         fclose(fp);
      }
   }
   return (st == Solve_Succeeded || st == Solved_To_Acceptable_Level) ? 0 : 1;
}
