// capi.cu -- extern "C" boundary of libmjb200.so (see include/mjb200.h for the reference interfaces each entry replaces).
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
using std::min;
#include <string>

#include "../../include/mjb200.h"
#include "mjb_types.cuh"

struct mjbModel {
  ModelDev dev;
  bool finalized;
};
struct mjbData {
  DataDev dev;
  bool finalized;
  size_t smem[6];
  // step pipelining over two world halves on two internal streams (overlaps each kernel's partial last wave with the
  // other half's kernels; worlds never interact, so the halves are independent apart from the shared contact-pool counter)
  cudaStream_t aux[8];
  cudaEvent_t ev_fork, ev_join[8];
  int nsplit;
  cudaStream_t sol_aux[8];        // solver row-capacity classes: second class of each world range runs here
  cudaEvent_t sol_fork[8], sol_join[8];
  // fwd_velocity / fwd_actuation / fwd_acceleration need nothing collision or make_constraint write, so inside a world range
  // k_velocity can run on its own stream next to k_collision -> k_constraint and be joined before the solver (MJB_FORK=1; default serial)
  cudaStream_t vel_aux[8];
  cudaEvent_t vel_fork[8], vel_join[8];
  bool fork_velocity;
  float* rk;  // Runge-Kutta scratch, (nworld, nq + 3 nv + 2 na); allocated by mjb_data_finalize for RK4 models only
};

namespace {
thread_local std::string g_err;
thread_local int g_launches = 0;
int fail(const std::string& s) { g_err = s; return -1; }
int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  return fail(std::string(what) + ": " + cudaGetErrorString(e));
}
constexpr size_t kMaxSmem = 227 * 1024;
}  // namespace

extern "C" {

const char* mjb_last_error(void) { return g_err.c_str(); }
const char* mjb_version(void) { return "mjb200 0.1 (sm_90a)"; }
int mjb_last_launch_count(void) { return g_launches; }

mjbModel* mjb_model_create(void) {
  mjbModel* m = new mjbModel();
  memset(&m->dev, 0, sizeof(ModelDev));
  m->finalized = false;
  return m;
}
void mjb_model_destroy(mjbModel* m) { delete m; }

int mjb_model_set_int(mjbModel* m, const char* name, int v) {
#define X(n) if (!strcmp(name, #n)) { m->dev.n = v; return 0; }
  MJB_MODEL_INTS(X)
#undef X
  return fail(std::string("unknown model int field: ") + name);
}
int mjb_model_set_float(mjbModel* m, const char* name, float v) {
#define X(n) if (!strcmp(name, #n)) { m->dev.n = v; return 0; }
  MJB_MODEL_FLOATS(X)
#undef X
  return fail(std::string("unknown model float field: ") + name);
}
int mjb_model_set_array_batched(mjbModel* m, const char* name, const void* p, int nbatch, int batch_stride) {
  if (nbatch < 1) return fail(std::string("nbatch must be >= 1: ") + name);
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("integer Model tables are shared by all worlds (not batched): ") + name); m->dev.n = (const int*)p; return 0; }
  MJB_MODEL_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->dev.n = (const float*)p; m->dev.nb_##n = nbatch; m->dev.bs_##n = batch_stride; goto done; }
  MJB_MODEL_FARRS(X)
#undef X
  return fail(std::string("unknown model array field: ") + name);
done:
  m->dev.batched = 0;
#define X(n) if (m->dev.nb_##n > 1) m->dev.batched = 1;
  MJB_MODEL_FARRS(X)
#undef X
  return 0;
}
int mjb_model_set_array(mjbModel* m, const char* name, const void* p, int nbatch) {
  if (nbatch != 1) return fail(std::string("use mjb_model_set_array_batched (needs the per-entry stride) for a per-world field: ") + name);
  return mjb_model_set_array_batched(m, name, p, 1, 0);
}
int mjb_model_finalize(mjbModel* m) {
#define X(n) if (!m->dev.n) return fail(std::string("model array not set: ") + #n);
  MJB_MODEL_IARRS(X)
  MJB_MODEL_FARRS(X)
#undef X
  if (m->dev.nv <= 0 || m->dev.nbody <= 0) return fail("model has no dofs/bodies");
  if (m->dev.solver != SOL_NEWTON && m->dev.solver != SOL_CG) return fail("only the Newton and CG solvers are implemented");
  if (m->dev.cone != CONE_PYRAMIDAL && m->dev.cone != CONE_ELLIPTIC) return fail("unknown friction cone type");
  if (m->dev.integrator != INT_EULER && m->dev.integrator != INT_RK4 && m->dev.integrator != INT_IMPLICITFAST && m->dev.integrator != INT_IMPLICIT) return fail("unknown integrator");
  m->finalized = true;
  return 0;
}

mjbData* mjb_data_create(int nworld, int nconmax, int naconmax, int njmax, int njmax_pad, int nv_pad) {
  mjbData* d = new mjbData();
  memset(&d->dev, 0, sizeof(DataDev));
  d->dev.nworld = nworld; d->dev.nconmax = nconmax; d->dev.naconmax = naconmax;
  d->dev.njmax = njmax; d->dev.njmax_pad = njmax_pad; d->dev.nv_pad = nv_pad;
  d->dev.w0 = 0; d->dev.wn = nworld;
  d->finalized = false;
  d->nsplit = 1;
  d->rk = nullptr;
  return d;
}
void mjb_data_destroy(mjbData* d) {
  if (!d) return;
  if (d->dev.world_conadr) cudaFree(d->dev.world_conadr);
  if (d->dev.world_ncon) cudaFree(d->dev.world_ncon);
  if (d->dev.imp_qacc) cudaFree(d->dev.imp_qacc);
  if (d->dev.sol_list) cudaFree(d->dev.sol_list);
  if (d->dev.sol_count) {
    cudaFree(d->dev.sol_count);
    for (int i = 0; i < 8; i++) { cudaStreamDestroy(d->sol_aux[i]); cudaEventDestroy(d->sol_fork[i]); cudaEventDestroy(d->sol_join[i]); }
    for (int i = 0; i < 8; i++) { cudaStreamDestroy(d->vel_aux[i]); cudaEventDestroy(d->vel_fork[i]); cudaEventDestroy(d->vel_join[i]); }
  }
  if (d->rk) cudaFree(d->rk);
  if (d->nsplit > 1) {
    for (int i = 0; i < d->nsplit; i++) { cudaStreamDestroy(d->aux[i]); cudaEventDestroy(d->ev_join[i]); }
    cudaEventDestroy(d->ev_fork);
  }
  delete d;
}
int mjb_data_set_int(mjbData* d, const char* name, int v) {
  if (!strcmp(name, "njmax_nnz")) { d->dev.njmax_nnz = v; return 0; }
  return fail(std::string("unknown data int field: ") + name);
}
int mjb_data_set_array(mjbData* d, const char* name, void* p) {
#define X(n) if (!strcmp(name, #n)) { d->dev.n = (float*)p; return 0; }
  MJB_DATA_FARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { d->dev.n = (int*)p; return 0; }
  MJB_DATA_IARRS(X)
#undef X
  return fail(std::string("unknown data array field: ") + name);
}
int mjb_data_finalize(mjbData* d, const mjbModel* m) {
  if (!m || !m->finalized) return fail("model not finalized");
#define X(n) if (!d->dev.n) return fail(std::string("data array not set: ") + #n);
  MJB_DATA_FARRS(X)
  MJB_DATA_IARRS(X)
#undef X
  if (d->dev.nv_pad < m->dev.nv) return fail("nv_pad < nv");
  // nv > 32 solver: Jacobian rows staged in shared memory.  0 (rows are read through L2) by default: the smaller per-world slice lets
  // more worlds share an SM
  { const char* e = getenv("MJB_JCAP"); d->dev.jcap = e ? atoi(e) : 0; if (d->dev.jcap < 0) d->dev.jcap = 0; }
  if (check(cudaMalloc(&d->dev.world_conadr, sizeof(int) * (size_t)d->dev.nworld), "cudaMalloc(world_conadr)")) return -1;
  if (check(cudaMalloc(&d->dev.world_ncon, sizeof(int) * (size_t)d->dev.nworld), "cudaMalloc(world_ncon)")) return -1;
  if (check(cudaMemset(d->dev.world_conadr, 0, sizeof(int) * (size_t)d->dev.nworld), "memset")) return -1;
  if (check(cudaMemset(d->dev.world_ncon, 0, sizeof(int) * (size_t)d->dev.nworld), "memset")) return -1;
  // always there (nworld x nv floats), so that switching Option.integrator to the fully implicit one needs no allocation inside a graph capture
  if (check(cudaMalloc(&d->dev.imp_qacc, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nv > 0 ? m->dev.nv : 1)), "cudaMalloc(imp_qacc)")) return -1;
  if (check(cudaMalloc(&d->dev.sol_list, sizeof(int) * 2 * (size_t)d->dev.nworld), "cudaMalloc(sol_list)")) return -1;
  if (check(cudaMalloc(&d->dev.sol_count, sizeof(int) * 16), "cudaMalloc(sol_count)")) return -1;
  if (check(cudaMemset(d->dev.sol_count, 0, sizeof(int) * 16), "memset")) return -1;
  for (int i = 0; i < 8; i++) {
    if (check(cudaStreamCreateWithFlags(&d->sol_aux[i], cudaStreamNonBlocking), "cudaStreamCreate")) return -1;
    if (check(cudaEventCreateWithFlags(&d->sol_fork[i], cudaEventDisableTiming), "cudaEventCreate")) return -1;
    if (check(cudaEventCreateWithFlags(&d->sol_join[i], cudaEventDisableTiming), "cudaEventCreate")) return -1;
  }
  d->dev.sol_stream = d->sol_aux[0]; d->dev.sol_fork = d->sol_fork[0]; d->dev.sol_join = d->sol_join[0];
  for (int i = 0; i < 8; i++) {
    if (check(cudaStreamCreateWithFlags(&d->vel_aux[i], cudaStreamNonBlocking), "cudaStreamCreate")) return -1;
    if (check(cudaEventCreateWithFlags(&d->vel_fork[i], cudaEventDisableTiming), "cudaEventCreate")) return -1;
    if (check(cudaEventCreateWithFlags(&d->vel_join[i], cudaEventDisableTiming), "cudaEventCreate")) return -1;
  }
  {
    // equality rows read cvel / cdof_dot of the previous step (constraint.py:1085-1117 uses them as they stand when make_constraint
    // runs), which k_velocity overwrites: models with equalities keep the serial chain
    const char* e = getenv("MJB_FORK");
    // off by default: both branches are shared-memory bound, so running them side by side does not raise the number of resident
    // warps; MJB_FORK=1 enables it (bit-identical results, tested)
    d->fork_velocity = (e ? atoi(e) != 0 : false) && m->dev.neq == 0 && d->dev.nworld >= 1024;
  }
  if (m->dev.integrator == INT_RK4 && !d->rk &&
      check(cudaMalloc(&d->rk, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nq + 3 * m->dev.nv + 2 * m->dev.na + 1)), "cudaMalloc(rk)")) return -1;
  d->smem[0] = smem_position(m->dev); d->smem[1] = smem_collision(m->dev, d->dev); d->smem[2] = smem_constraint(m->dev, d->dev);
  d->smem[3] = smem_velocity(m->dev); d->smem[4] = smem_solver(m->dev, d->dev); d->smem[5] = smem_integrate(m->dev);
  static const char* names[6] = {"position", "collision", "constraint", "velocity", "solver", "integrate"};
  for (int i = 0; i < 6; i++)
    if (d->smem[i] > kMaxSmem) {
      char buf[160];
      snprintf(buf, sizeof buf, "%s kernel needs %zu B of shared memory per block (> %zu): model/njmax too large for this version", names[i], d->smem[i], kMaxSmem);
      return fail(buf);
    }
  {
    const char* e = getenv("MJB_SPLIT");
    const int want = e ? atoi(e) : 2;
    if (want >= 2 && d->dev.nworld >= 1024) {
      const int ns = want > 8 ? 8 : want;
      for (int i = 0; i < ns; i++) {
        if (check(cudaStreamCreateWithFlags(&d->aux[i], cudaStreamNonBlocking), "cudaStreamCreate")) return -1;
        if (check(cudaEventCreateWithFlags(&d->ev_join[i], cudaEventDisableTiming), "cudaEventCreate")) return -1;
      }
      if (check(cudaEventCreateWithFlags(&d->ev_fork, cudaEventDisableTiming), "cudaEventCreate")) return -1;
      d->nsplit = ns;
    }
  }
  d->finalized = true;
  return 0;
}

#define MJB_ENTER()                                                                 \
  if (!m || !d || !m->finalized || !d->finalized) return fail("model/data not finalized"); \
  cudaStream_t s = (cudaStream_t)stream;                                             \
  g_launches = 0;
#define MJB_LAUNCH(call, n) do { if (check((call), #call)) return -1; g_launches += (n); } while (0)

int mjb_kinematics(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_KINEMATICS, s), 1); return 0; }
int mjb_com_pos(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_COM_POS, s), 1); return 0; }
int mjb_camlight(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_CAMLIGHT, s), 1); return 0; }
int mjb_crb(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_CRB, s), 1); return 0; }
int mjb_transmission(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_TRANSMISSION, s), 1); return 0; }
int mjb_collision(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(reset_contact_counters(d->dev, s), 0); MJB_LAUNCH(launch_collision(m->dev, d->dev, s), 1); return 0; }
int mjb_make_constraint(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(launch_constraint(m->dev, d->dev, s), 1);
  if (d->dev.njmax_nnz > 0) MJB_LAUNCH(launch_efc_csr(m->dev, d->dev, s), 1);
  return 0;
}
int mjb_fwd_velocity(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_VELOCITY, s), 1); return 0; }
int mjb_fwd_actuation(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_ACTUATION, s), 1); return 0; }
int mjb_fwd_acceleration(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_ACCELERATION, s), 1); return 0; }
int mjb_factor_m(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_FACTOR_ONLY, s), 1); return 0; }
int mjb_com_vel(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_COMVEL, s), 1); return 0; }
int mjb_passive(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_PASSIVE, s), 1); return 0; }
int mjb_rne(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_RNE, s), 1); return 0; }
int mjb_solve_m(const mjbModel* m, mjbData* d, float* x, const float* y, void* stream) {
  MJB_ENTER();
  if (!x || !y) return fail("mjb_solve_m: null vector");
  MJB_LAUNCH(launch_solve_m(m->dev, d->dev, x, y, s), 1);
  return 0;
}
int mjb_mul_m(const mjbModel* m, mjbData* d, float* res, const float* vec, void* stream) {
  MJB_ENTER();
  if (!res || !vec) return fail("mjb_mul_m: null vector");
  MJB_LAUNCH(launch_mul_m(m->dev, d->dev, res, vec, s), 1);
  return 0;
}
int mjb_contact_force(const mjbModel* m, mjbData* d, const int* contact_ids, int n, int to_world_frame, float* force, void* stream) {
  MJB_ENTER();
  if (n > 0 && (!contact_ids || !force)) return fail("mjb_contact_force: null array");
  MJB_LAUNCH(launch_contact_force(m->dev, d->dev, contact_ids, n, to_world_frame, force, s), 1);
  return 0;
}
int mjb_sensor_pos(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_sensor(m->dev, d->dev, 1, s), 1); return 0; }
int mjb_sensor_vel(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_sensor(m->dev, d->dev, 2, s), 1); return 0; }
int mjb_sensor_acc(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_sensor(m->dev, d->dev, 4, s), 1); return 0; }
int mjb_solve(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_solver(m->dev, d->dev, s), solver_launch_count(m->dev, d->dev)); return 0; }
int mjb_euler(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_integrate(m->dev, d->dev, INT_EULER, s), 1); return 0; }
int mjb_implicit(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  if (m->dev.integrator != INT_IMPLICIT && m->dev.integrator != INT_IMPLICITFAST) return fail("mjb_implicit: the model's integrator is Euler / RK4 (the factor-and-solve scratch is sized by the integrator the model was created with)");
  if (m->dev.integrator == INT_IMPLICIT && smem_implicit(m->dev) > kMaxSmem) return fail("implicit integrator: the velocity-derivative scratch (18 x nbody x 32 floats) exceeds one block's shared memory");
  MJB_LAUNCH(launch_integrate(m->dev, d->dev, m->dev.integrator == INT_IMPLICIT ? INT_IMPLICIT : INT_IMPLICITFAST, s), m->dev.integrator == INT_IMPLICIT ? 2 : 1);
  return 0;
}

// which stages a pipeline call runs
enum { RUN_POSITION = 1, RUN_VELOCITY = 2, RUN_SOLVER = 4, RUN_EULER = 8 };

static int chain(const mjbModel* m, const mjbData* d, const DataDev& dd, int what, cudaStream_t s) {
  const bool fork = d->fork_velocity && (what & RUN_POSITION) && (what & RUN_VELOCITY);
  const int h = dd.split_id;
  if (what & RUN_POSITION) {
    // forward.py:635-677 with factorize=False: kinematics, com_pos, camlight, crb, collision, make_constraint, transmission
    MJB_LAUNCH(launch_position(m->dev, dd, STG_KINEMATICS | STG_COM_POS | STG_CAMLIGHT | STG_CRB | STG_TRANSMISSION, s), 1);
    if (fork) {
      if (check(cudaEventRecord(d->vel_fork[h], s), "cudaEventRecord")) return -1;
      if (check(cudaStreamWaitEvent(d->vel_aux[h], d->vel_fork[h], 0), "cudaStreamWaitEvent")) return -1;
      MJB_LAUNCH(launch_velocity(m->dev, dd, STG_VELOCITY | STG_ACTUATION | STG_ACCELERATION, d->vel_aux[h]), 1);
      if (check(cudaEventRecord(d->vel_join[h], d->vel_aux[h]), "cudaEventRecord")) return -1;
    }
    MJB_LAUNCH(launch_collision(m->dev, dd, s), 1);
    MJB_LAUNCH(launch_constraint(m->dev, dd, s), 1);
    if (dd.njmax_nnz > 0) MJB_LAUNCH(launch_efc_csr(m->dev, dd, s), 1);  // sparse models: the reference's CSR arrays next to the dense rows
  }
  if (fork) { if (check(cudaStreamWaitEvent(s, d->vel_join[h], 0), "cudaStreamWaitEvent")) return -1; }
  else if (what & RUN_VELOCITY) MJB_LAUNCH(launch_velocity(m->dev, dd, STG_VELOCITY | STG_ACTUATION | STG_ACCELERATION, s), 1);
  if (what & RUN_SOLVER) MJB_LAUNCH(launch_solver(m->dev, dd, s), solver_launch_count(m->dev, dd));
  // sensors of all three stages in one launch after the solver (forward.py:1350-1365 interleaves them; their inputs are final by now)
  if ((what & RUN_SOLVER) && m->dev.nsensor > 0) MJB_LAUNCH(launch_sensor(m->dev, dd, 7, s), 1);
  if (what & RUN_EULER) {
    if (m->dev.integrator == INT_IMPLICIT && smem_implicit(m->dev) > kMaxSmem) return fail("implicit integrator: the velocity-derivative scratch (18 x nbody x 32 floats) exceeds one block's shared memory");
    MJB_LAUNCH(launch_integrate(m->dev, dd, -1, s), m->dev.integrator == INT_IMPLICIT ? 2 : 1);
  }
  return 0;
}

static int pipeline(const mjbModel* m, mjbData* d, int what, cudaStream_t s) {
  if (what & RUN_POSITION) MJB_LAUNCH(reset_contact_counters(d->dev, s), 0);
  if (d->nsplit < 2) return chain(m, d, d->dev, what, s);
  // fork: both halves wait for everything queued on the caller's stream, run their own kernel chain, and are joined back
  if (check(cudaEventRecord(d->ev_fork, s), "cudaEventRecord")) return -1;
  const int part = (d->dev.nworld + d->nsplit - 1) / d->nsplit;
  for (int h = 0; h < d->nsplit; h++) {
    DataDev dd = d->dev;
    dd.w0 = h * part;
    dd.wn = min(part, d->dev.nworld - dd.w0);
    dd.split_id = h;
    dd.sol_stream = d->sol_aux[h]; dd.sol_fork = d->sol_fork[h]; dd.sol_join = d->sol_join[h];
    if (dd.wn <= 0) break;
    if (check(cudaStreamWaitEvent(d->aux[h], d->ev_fork, 0), "cudaStreamWaitEvent")) return -1;
    if (chain(m, d, dd, what, d->aux[h])) return -1;
    if (check(cudaEventRecord(d->ev_join[h], d->aux[h]), "cudaEventRecord")) return -1;
    if (check(cudaStreamWaitEvent(s, d->ev_join[h], 0), "cudaStreamWaitEvent")) return -1;
  }
  return 0;
}
int mjb_fwd_position(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); return pipeline(m, d, RUN_POSITION, s); }
int mjb_forward(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); return pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER, s); }
// forward.py:523-555 rungekutta4, called after forward(): three more forward() evaluations with the state bookkeeping in between
static int rk4_after_forward(const mjbModel* m, mjbData* d, cudaStream_t s) {
  if (!d->rk) return fail("Runge-Kutta scratch missing: data was finalized against a model whose integrator is not RK4");
  for (int stage = 0; stage < 4; stage++) {
    if (stage > 0 && pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER, s)) return -1;
    MJB_LAUNCH(launch_rk_stage(m->dev, d->dev, d->rk, stage, s), 1);
  }
  return 0;
}
int mjb_rungekutta4(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); return rk4_after_forward(m, d, s); }
int mjb_step(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  if (m->dev.integrator == INT_RK4) {
    if (pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER, s)) return -1;
    return rk4_after_forward(m, d, s);
  }
  return pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER | RUN_EULER, s);
}
int mjb_step_profile(const mjbModel* m, mjbData* d, void* stream, float* ms_out) {
  // one step with a CUDA event pair around every kernel; synchronises (profiling aid, not the hot path)
  MJB_ENTER();
  cudaEvent_t ev[7];
  for (int i = 0; i < 7; i++) if (check(cudaEventCreate(&ev[i]), "cudaEventCreate")) return -1;
  cudaEventRecord(ev[0], s);
  MJB_LAUNCH(launch_position(m->dev, d->dev, STG_KINEMATICS | STG_COM_POS | STG_CAMLIGHT | STG_CRB | STG_TRANSMISSION, s), 1);
  cudaEventRecord(ev[1], s);
  MJB_LAUNCH(reset_contact_counters(d->dev, s), 0);
  MJB_LAUNCH(launch_collision(m->dev, d->dev, s), 1);
  cudaEventRecord(ev[2], s);
  MJB_LAUNCH(launch_constraint(m->dev, d->dev, s), 1);
  cudaEventRecord(ev[3], s);
  MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_VELOCITY | STG_ACTUATION | STG_ACCELERATION, s), 1);
  cudaEventRecord(ev[4], s);
  MJB_LAUNCH(launch_solver(m->dev, d->dev, s), 1);
  cudaEventRecord(ev[5], s);
  MJB_LAUNCH(launch_integrate(m->dev, d->dev, -1, s), 1);
  cudaEventRecord(ev[6], s);
  if (check(cudaEventSynchronize(ev[6]), "cudaEventSynchronize")) return -1;
  for (int i = 0; i < 6; i++) cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]);
  for (int i = 0; i < 7; i++) cudaEventDestroy(ev[i]);
  return 0;
}
int mjb_ctrl_noise(const mjbModel* m, mjbData* d, const float* ctrl_center, int step, float noise_std, float noise_rate, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(launch_ctrl_noise(m->dev, d->dev, ctrl_center, step, noise_std, noise_rate, s), 1);
  return 0;
}

}  // extern "C"
