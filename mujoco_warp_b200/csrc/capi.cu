// capi.cu -- extern "C" boundary of libmjb200.so (see include/mjb200.h for the reference interfaces each entry replaces).
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
using std::min;
#include <string>

#include "../../include/mjb200.h"
#include "mjb_launch.cuh"
#include "mjb_types.cuh"

struct mjbModel {
  ModelDev dev;
  FluidDev fluid;  // qfrc_fluid stays null here: it is the Data's (fluid() below)
  SensorCollisionDev sc;
  SensorContactDev scon;  // the <contact> sensors and Option.contact_sensor_maxmatch
  RangefinderDev rf;      // the rangefinder sensors
  SetConstDev setc;  // actuator_acc0 and the meaninertia output, bound by name; qpos_save stays null here (the Data's)
  EnergyDev en;      // the energy sensors; energy stays null here (the Data's: energy() below)
  HistoryDev hist;   // the delay fields; history and ctrl_delayed stay null here (the Data's: history() below)
  MeshClipDev mclip;  // npolygonmax / nmeshdegmax; nslot and scratch stay zero here (the Data's: mesh_clip() below)
  bool finalized;
};
struct mjbData {
  DataDev dev;
  bool finalized;
  // step pipelining over two world halves on two internal streams (overlaps each kernel's partial last wave with the
  // other half's kernels; worlds never interact, so the halves are independent apart from the shared contact-pool counter)
  cudaStream_t aux[8];
  cudaEvent_t ev_fork, ev_join[8];
  int nsplit;
  float* rk;  // Runge-Kutta scratch, (nworld, nq + 3 nv + 2 na); allocated by mjb_data_finalize for RK4 models only
  // inverse dynamics (k_inverse.cu takes them as arguments: DataDev stays as the other kernels know it)
  float* qfrc_inverse;  // Data.qfrc_inverse, (nworld, nv), bound by name like the DataDev arrays
  float* inv_qacc;      // (nworld, nv) continuous-time acceleration of discrete inverse dynamics, read by its sensor launch
  float* qfrc_fluid;    // Data.qfrc_fluid, (nworld, nv), bound by name; passed to the fluid kernels in FluidDev
  float* qpos_save;     // (nworld, nq) d.qpos while mjb_set_const runs the position stages at qpos0 / qpos_spring
  float* energy;        // Data.energy, (nworld, 2), bound by name; passed to k_energy in EnergyDev
  float* history;       // Data.history, (nworld, nhistory), bound by name; passed to k_history in HistoryDev
  float* ctrl_delayed;  // (nworld, nu) the delayed ctrl the actuation stage reads; allocated for models with actuator delays only
  int mclip_nslot;      // slices per world of mclip_scratch
  float* mclip_scratch;  // the mesh multi-contact scratch (MeshClipDev); allocated for models past the fixed buffers only
};

namespace {
thread_local std::string g_err;
int fail(const std::string& s) { g_err = s; return -1; }
int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  return fail(std::string(what) + ": " + cudaGetErrorString(e));
}
constexpr size_t kMaxSmem = 227 * 1024;
}  // namespace

// The fluid fields of a model bound to a Data's qfrc_fluid
static FluidDev fluid(const mjbModel* m, const mjbData* d) { FluidDev f = m->fluid; f.qfrc_fluid = d->qfrc_fluid; return f; }
// The energy sensors of a model bound to a Data's energy
static EnergyDev energy(const mjbModel* m, const mjbData* d) { EnergyDev e = m->en; e.energy = d->energy; return e; }
// The delay fields of a model bound to a Data's history buffers
static HistoryDev history(const mjbModel* m, const mjbData* d) { HistoryDev h = m->hist; h.history = d->history; h.ctrl_delayed = d->ctrl_delayed; return h; }
// The mesh multi-contact sizes of a model bound to a Data's scratch; models with such hulls run the CCD_MESH = 2 kernels
static MeshClipDev mesh_clip(const mjbModel* m, const mjbData* d) { MeshClipDev c = m->mclip; c.nslot = d->mclip_nslot; c.scratch = d->mclip_scratch; return c; }
static bool mesh_large(const mjbModel* m) { return m->dev.nmesh > 0 && mesh_clip_large(m->mclip.npolygonmax, m->mclip.nmeshdegmax); }
// scratch slices per world: k_collision's GJK / EPA lanes (4), or the collision-sensor kernel's EPA slots when it has more
static int mesh_clip_slots(const mjbModel* m) { return std::max(4, std::min(32, m->sc.nsensorcollision_ccd)); }
static cudaError_t collision(const mjbModel* m, const mjbData* d, const DataDev& dd, cudaStream_t s) {
  return mesh_large(m) ? launch_collision_mesh_large(m->dev, dd, mesh_clip(m, d), s) : launch_collision(m->dev, dd, s);
}

extern "C" {

const char* mjb_last_error(void) { return g_err.c_str(); }
const char* mjb_version(void) { return "mjb200 0.1 (sm_90a)"; }
int mjb_last_launch_count(void) { return g_launches; }

mjbModel* mjb_model_create(void) {
  mjbModel* m = new mjbModel();
  memset(&m->dev, 0, sizeof(ModelDev));
  memset(&m->fluid, 0, sizeof(FluidDev));
  memset(&m->sc, 0, sizeof(SensorCollisionDev));
  memset(&m->scon, 0, sizeof(SensorContactDev));
  memset(&m->rf, 0, sizeof(RangefinderDev));
  memset(&m->setc, 0, sizeof(SetConstDev));
  memset(&m->en, 0, sizeof(EnergyDev));
  memset(&m->hist, 0, sizeof(HistoryDev));
  memset(&m->mclip, 0, sizeof(MeshClipDev));
  m->finalized = false;
  return m;
}
void mjb_model_destroy(mjbModel* m) { delete m; }

int mjb_model_set_int(mjbModel* m, const char* name, int v) {
#define X(n) if (!strcmp(name, #n)) { m->dev.n = v; return 0; }
  MJB_MODEL_INTS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->fluid.n = v; return 0; }
  MJB_FLUID_INTS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->sc.n = v; return 0; }
  MJB_SENSCOL_INTS(X)
#undef X
  if (!strcmp(name, "contact_sensor_maxmatch")) {
    SensorContactDev c = m->scon;
    c.contact_sensor_maxmatch = v;
    if (v < 1 || smem_sensor_contact(c) > kMaxSmem)
      return fail("contact_sensor_maxmatch must be in [1, " + std::to_string(kMaxSmem / smem_sensor_contact(SensorContactDev{0, 1, nullptr, nullptr})) + "], got " + std::to_string(v));
    m->scon.contact_sensor_maxmatch = v;
    return 0;
  }
  if (!strcmp(name, "nsensorcontact")) { m->scon.nsensorcontact = v; return 0; }
#define X(n) if (!strcmp(name, #n)) { m->rf.n = v; return 0; }
  MJB_RANGEFINDER_INTS(X)
#undef X
  if (!strcmp(name, "sensor_extra")) { m->dev.sensor_extra = v; return 0; }
#define X(n) if (!strcmp(name, #n)) { m->en.n = v; return 0; }
  MJB_ENERGY_INTS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->hist.n = v; return 0; }
  MJB_HISTORY_INTS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->mclip.n = v; return 0; }
  MJB_MESHCLIP_INTS(X)
#undef X
  return fail(std::string("unknown model int field: ") + name);
}
int mjb_model_set_float(mjbModel* m, const char* name, float v) {
#define X(n) if (!strcmp(name, #n)) { m->dev.n = v; return 0; }
  MJB_MODEL_FLOATS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { m->fluid.n = v; return 0; }
  MJB_FLUID_FLOATS(X)
#undef X
  return fail(std::string("unknown model float field: ") + name);
}
int mjb_model_set_array_batched(mjbModel* m, const char* name, const void* p, int nbatch, int batch_stride) {
  if (nbatch < 1) return fail(std::string("nbatch must be >= 1: ") + name);
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("integer Model tables are shared by all worlds (not batched): ") + name); m->dev.n = (const int*)p; return 0; }
  MJB_MODEL_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->fluid.n = (decltype(m->fluid.n))p; return 0; }
  MJB_FLUID_IARRS(X)
  MJB_FLUID_FARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->sc.n = (const int*)p; return 0; }
  MJB_SENSCOL_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->scon.n = (const int*)p; return 0; }
  MJB_SENSCON_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->rf.n = (const int*)p; return 0; }
  MJB_RANGEFINDER_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->en.n = (const int*)p; return 0; }
  MJB_ENERGY_IARRS(X)
#undef X
#define X(n) if (!strcmp(name, #n)) { if (nbatch != 1) return fail(std::string("shared by all worlds (not batched): ") + name); m->hist.n = (decltype(m->hist.n))p; return 0; }
  MJB_HISTORY_IARRS(X)
  MJB_HISTORY_FARRS(X)
#undef X
  // set_const writes actuator_acc0 through SetConstDev; the muscle actuators read it through ModelDev (below)
  if (!strcmp(name, "actuator_acc0")) { m->setc.actuator_acc0 = (float*)p; m->setc.nb_actuator_acc0 = nbatch; }
  if (!strcmp(name, "meaninertia")) {
    if (nbatch != 1) return fail("meaninertia is a Model scalar (not batched)");
    m->setc.meaninertia = (float*)p;
    return 0;
  }
  if (!strcmp(name, "cam_resolution")) { if (nbatch != 1) return fail("integer Model tables are shared by all worlds (not batched): cam_resolution"); m->dev.cam_resolution = (const int*)p; return 0; }
#define X(n) if (!strcmp(name, #n)) { m->dev.n = (const float*)p; m->dev.nb_##n = nbatch; m->dev.bs_##n = batch_stride; goto done; }
  MJB_MODEL_FARRS(X)
  MJB_MODEL_SENSOR_FARRS(X)
#undef X
  return fail(std::string("unknown model array field: ") + name);
done:
  m->dev.batched = 0;
#define X(n) if (m->dev.nb_##n > 1) m->dev.batched = 1;
  MJB_MODEL_FARRS(X)
  MJB_MODEL_SENSOR_FARRS(X)
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
  MJB_MODEL_SENSOR_FARRS(X)
  X(cam_resolution)
#undef X
#define X(n) if (!m->fluid.n) return fail(std::string("model array not set: ") + #n);
  MJB_FLUID_IARRS(X)
  MJB_FLUID_FARRS(X)
#undef X
#define X(n) if (!m->sc.n) return fail(std::string("model array not set: ") + #n);
  MJB_SENSCOL_IARRS(X)
#undef X
#define X(n) if (!m->scon.n) return fail(std::string("model array not set: ") + #n);
  MJB_SENSCON_IARRS(X)
#undef X
  if (m->scon.contact_sensor_maxmatch < 1) return fail("model int not set: contact_sensor_maxmatch");
#define X(n) if (!m->rf.n) return fail(std::string("model array not set: ") + #n);
  MJB_RANGEFINDER_IARRS(X)
#undef X
#define X(n) if (!m->en.n) return fail(std::string("model array not set: ") + #n);
  MJB_ENERGY_IARRS(X)
#undef X
#define X(n) if (!m->hist.n) return fail(std::string("model array not set: ") + #n);
  MJB_HISTORY_IARRS(X)
  MJB_HISTORY_FARRS(X)
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
  d->qfrc_inverse = nullptr;
  d->inv_qacc = nullptr;
  d->qfrc_fluid = nullptr;
  d->qpos_save = nullptr;
  d->energy = nullptr;
  d->history = nullptr;
  d->ctrl_delayed = nullptr;
  d->mclip_nslot = 0;
  d->mclip_scratch = nullptr;
  return d;
}
void mjb_data_destroy(mjbData* d) {
  if (!d) return;
  if (d->dev.world_conadr) cudaFree(d->dev.world_conadr);
  if (d->dev.world_ncon) cudaFree(d->dev.world_ncon);
  if (d->dev.imp_qacc) cudaFree(d->dev.imp_qacc);
  if (d->inv_qacc) cudaFree(d->inv_qacc);
  if (d->rk) cudaFree(d->rk);
  if (d->qpos_save) cudaFree(d->qpos_save);
  if (d->ctrl_delayed) cudaFree(d->ctrl_delayed);
  if (d->mclip_scratch) cudaFree(d->mclip_scratch);
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
  if (!strcmp(name, "qfrc_inverse")) { d->qfrc_inverse = (float*)p; return 0; }
  if (!strcmp(name, "qfrc_fluid")) { d->qfrc_fluid = (float*)p; return 0; }
  if (!strcmp(name, "energy")) { d->energy = (float*)p; return 0; }
  if (!strcmp(name, "history")) { d->history = (float*)p; return 0; }
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
  if (!d->qfrc_inverse) return fail("data array not set: qfrc_inverse");
  if (!d->qfrc_fluid) return fail("data array not set: qfrc_fluid");
  if (!d->energy) return fail("data array not set: energy");
  if (!d->history) return fail("data array not set: history");
  if (d->dev.nv_pad < m->dev.nv) return fail("nv_pad < nv");
  if (check(cudaMalloc(&d->dev.world_conadr, sizeof(int) * (size_t)d->dev.nworld), "cudaMalloc(world_conadr)")) return -1;
  if (check(cudaMalloc(&d->dev.world_ncon, sizeof(int) * (size_t)d->dev.nworld), "cudaMalloc(world_ncon)")) return -1;
  if (check(cudaMemset(d->dev.world_conadr, 0, sizeof(int) * (size_t)d->dev.nworld), "memset")) return -1;
  if (check(cudaMemset(d->dev.world_ncon, 0, sizeof(int) * (size_t)d->dev.nworld), "memset")) return -1;
  // always there (nworld x nv floats), so that switching Option.integrator to the fully implicit one needs no allocation inside a graph capture
  if (check(cudaMalloc(&d->dev.imp_qacc, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nv > 0 ? m->dev.nv : 1)), "cudaMalloc(imp_qacc)")) return -1;
  // likewise always there, so that enabling discrete inverse dynamics (Option.enableflags) needs no allocation either
  if (!d->inv_qacc && check(cudaMalloc(&d->inv_qacc, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nv > 0 ? m->dev.nv : 1)), "cudaMalloc(inv_qacc)")) return -1;
  // set_const's save buffer, so that mjb_set_const allocates nothing (and can be captured in a graph)
  if (!d->qpos_save && check(cudaMalloc(&d->qpos_save, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nq > 0 ? m->dev.nq : 1)), "cudaMalloc(qpos_save)")) return -1;
  if (m->hist.nactuator_history > 0 && !d->ctrl_delayed &&
      check(cudaMalloc(&d->ctrl_delayed, sizeof(float) * (size_t)d->dev.nworld * (size_t)m->dev.nu), "cudaMalloc(ctrl_delayed)")) return -1;
  if (m->dev.integrator == INT_RK4 && !d->rk &&
      check(cudaMalloc(&d->rk, sizeof(float) * (size_t)d->dev.nworld * (size_t)(m->dev.nq + 3 * m->dev.nv + 2 * m->dev.na + 1)), "cudaMalloc(rk)")) return -1;
  const size_t smem[6] = {smem_position(m->dev, d->dev), smem_collision(m->dev, d->dev), smem_constraint(m->dev, d->dev),
                          smem_velocity(m->dev, d->dev, fluid(m, d)), smem_solver(m->dev, d->dev),    smem_integrate(m->dev)};
  static const char* names[6] = {"position", "collision", "constraint", "velocity", "solver", "integrate"};
  for (int i = 0; i < 6; i++)
    if (smem[i] > kMaxSmem) {
      char buf[160];
      snprintf(buf, sizeof buf, "%s kernel needs %zu B of shared memory per block (> %zu): model/njmax too large for this version", names[i], smem[i], kMaxSmem);
      return fail(buf);
    }
  if (smem_sensor_collision(m->sc) > kMaxSmem) {
    char buf[200];
    snprintf(buf, sizeof buf, "collision-sensor kernel needs %zu B of shared memory per block (> %zu): too many sensor geom pairs or GJK / EPA iterations",
             smem_sensor_collision(m->sc), kMaxSmem);
    return fail(buf);
  }
  if (mesh_large(m) && !d->mclip_scratch) {
    d->mclip_nslot = mesh_clip_slots(m);
    const size_t bytes = sizeof(float) * (size_t)d->dev.nworld * (size_t)d->mclip_nslot * (size_t)mesh_clip_words(m->mclip);
    if (cudaMalloc(&d->mclip_scratch, bytes) != cudaSuccess) {
      cudaGetLastError();
      d->mclip_scratch = nullptr;
      char buf[240];
      snprintf(buf, sizeof buf, "collision kernel needs %zu B of global scratch for the mesh multi-contact (%d worlds x %d slices x %d floats; npolygonmax %d, nmeshdegmax %d)",
               bytes, d->dev.nworld, d->mclip_nslot, mesh_clip_words(m->mclip), m->mclip.npolygonmax, m->mclip.nmeshdegmax);
      return fail(buf);
    }
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
#define MJB_LAUNCH(call) do { if (check((call), #call)) return -1; } while (0)

// The Data the actuation stage reads for dd's world range (forward.py:1161-1165): with actuator delays its ctrl is the delayed one,
// which k_history_ctrl_read writes first.  Every other kernel keeps reading d.ctrl.
static int actuation_data(const mjbModel* m, const mjbData* d, const DataDev& dd, cudaStream_t s, DataDev* out) {
  *out = dd;
  if (m->hist.nactuator_history == 0) return 0;
  out->ctrl = d->ctrl_delayed;
  return check(launch_history_ctrl_read(m->dev, dd, history(m, d), s), "launch_history_ctrl_read");
}
// The actuator buffers take d.ctrl at d.time before the integrator advances it (forward.py:320, _advance)
static cudaError_t history_ctrl_insert(const mjbModel* m, const mjbData* d, const DataDev& dd, cudaStream_t s) {
  return m->hist.nactuator_history > 0 ? launch_history_ctrl_insert(m->dev, dd, history(m, d), s) : cudaSuccess;
}
// The sensors of `stages` with a buffer report their delayed / held value and record the fresh one (sensor.py:956, :1502, :2765)
static cudaError_t history_sensor(const mjbModel* m, const mjbData* d, const DataDev& dd, int stages, cudaStream_t s) {
  if (m->hist.nsensor_history == 0 || (m->dev.disableflags & DSBL_SENSOR)) return cudaSuccess;
  return launch_history_sensor(m->dev, dd, history(m, d), stages, s);
}

int mjb_kinematics(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_KINEMATICS, s)); return 0; }
int mjb_com_pos(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_COM_POS, s)); return 0; }
int mjb_camlight(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_CAMLIGHT, s)); return 0; }
int mjb_crb(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_CRB, s)); return 0; }
int mjb_transmission(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_position(m->dev, d->dev, STG_TRANSMISSION, s)); return 0; }
int mjb_collision(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(reset_contact_counters(d->dev, s)); MJB_LAUNCH(collision(m, d, d->dev, s)); return 0; }
int mjb_make_constraint(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(launch_constraint(m->dev, d->dev, s));
  if (d->dev.njmax_nnz > 0) MJB_LAUNCH(launch_efc_csr(m->dev, d->dev, s));
  return 0;
}
int mjb_fwd_velocity(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_VELOCITY, s, fluid(m, d))); return 0; }
int mjb_fwd_actuation(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  DataDev da;
  if (actuation_data(m, d, d->dev, s, &da)) return -1;
  MJB_LAUNCH(launch_velocity(m->dev, da, STG_ACTUATION, s, fluid(m, d)));
  return 0;
}
int mjb_fwd_acceleration(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_ACCELERATION, s, fluid(m, d))); return 0; }
int mjb_factor_m(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_FACTOR_ONLY, s, fluid(m, d))); return 0; }
int mjb_com_vel(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_COMVEL, s, fluid(m, d))); return 0; }
int mjb_passive(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_PASSIVE, s, fluid(m, d))); return 0; }
int mjb_rne(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_velocity(m->dev, d->dev, STG_RNE, s, fluid(m, d))); return 0; }
int mjb_solve_m(const mjbModel* m, mjbData* d, float* x, const float* y, void* stream) {
  MJB_ENTER();
  if (!x || !y) return fail("mjb_solve_m: null vector");
  MJB_LAUNCH(launch_solve_m(m->dev, d->dev, x, y, s));
  return 0;
}
int mjb_mul_m(const mjbModel* m, mjbData* d, float* res, const float* vec, void* stream) {
  MJB_ENTER();
  if (!res || !vec) return fail("mjb_mul_m: null vector");
  MJB_LAUNCH(launch_mul_m(m->dev, d->dev, res, vec, s));
  return 0;
}
int mjb_contact_force(const mjbModel* m, mjbData* d, const int* contact_ids, int n, int to_world_frame, float* force, void* stream) {
  MJB_ENTER();
  if (n > 0 && (!contact_ids || !force)) return fail("mjb_contact_force: null array");
  MJB_LAUNCH(launch_contact_force(m->dev, d->dev, contact_ids, n, to_world_frame, force, s));
  return 0;
}
// smooth.py:1744 rne_postconstraint, :3614 subtree_vel, :4197 tendon; support.py:583 jac, :314 xfrc_accumulate; derivative.py:1117
// deriv_smooth_vel: one launch each over every world (none for tendon without tendons, nor for jac / xfrc_accumulate without dofs),
// whatever the model's sensors or DSBL_SENSOR say
int mjb_rne_postconstraint(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_rne_postconstraint(m->dev, d->dev, s)); return 0; }
int mjb_subtree_vel(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_subtree_vel(m->dev, d->dev, s)); return 0; }
int mjb_tendon(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_tendon(m->dev, d->dev, s)); return 0; }
int mjb_jac(const mjbModel* m, mjbData* d, float* jacp, float* jacr, const float* point, const int* body, void* stream) {
  MJB_ENTER();
  if (!point || !body) return fail("mjb_jac: null point / body array");
  MJB_LAUNCH(launch_jac(m->dev, d->dev, jacp, jacr, point, body, s));
  return 0;
}
int mjb_xfrc_accumulate(const mjbModel* m, mjbData* d, float* qfrc, void* stream) {
  MJB_ENTER();
  if (!qfrc) return fail("mjb_xfrc_accumulate: null qfrc");
  MJB_LAUNCH(launch_xfrc_accumulate(m->dev, d->dev, qfrc, s));
  return 0;
}
int mjb_deriv_smooth_vel(const mjbModel* m, mjbData* d, float* out, void* stream) {
  MJB_ENTER();
  if (!out) return fail("mjb_deriv_smooth_vel: null out");
  if (smem_deriv_smooth_vel(m->dev) > kMaxSmem) return fail("mjb_deriv_smooth_vel: the largest tree's block exceeds one block's shared memory");
  MJB_LAUNCH(launch_deriv_smooth_vel(m->dev, d->dev, out, s, fluid(m, d)));
  return 0;
}
int mjb_rays(const mjbModel* m, mjbData* d, const float* pnt, const float* vec, int nray, int pnt_nbatch, const int* geomgroup, int flg_static,
             const int* bodyexclude, float* dist, int* geomid, float* normal, void* stream) {
  MJB_ENTER();
  const int nworld = d->dev.nworld;
  if (nray < 0) return fail("mjb_rays: nray must be >= 0, got " + std::to_string(nray));
  if (pnt_nbatch != 1 && pnt_nbatch != nworld) return fail("mjb_rays: pnt_nbatch must be 1 or nworld (" + std::to_string(nworld) + "), got " + std::to_string(pnt_nbatch));
  if ((long long)nworld * nray > 0x7fffffffLL) return fail("mjb_rays: nworld * nray exceeds the int range");
  if (nray > 0 && (!pnt || !vec || !bodyexclude || !dist || !geomid || !normal)) return fail("mjb_rays: null array");
  MJB_LAUNCH(launch_ray(m->dev, d->dev, pnt, vec, nray, pnt_nbatch, geomgroup, flg_static, bodyexclude, dist, geomid, normal, s));
  return 0;
}
static int check_render(const mjbModel* m, const mjbData* d, const mjbRender* rc, const char* what) {
  if (!rc) return fail(std::string(what) + ": null render context");
  if (rc->ngeom < 0 || rc->ncam < 0 || rc->npixel < 0) return fail(std::string(what) + ": negative size in the render context");
  if (rc->ngeom > 0 && (!rc->geom_id || !rc->lower || !rc->upper)) return fail(std::string(what) + ": null geom table");
  if (smem_render(rc->ngeom) > kMaxSmem)
    return fail(std::string(what) + ": " + std::to_string(rc->ngeom) + " enabled geoms exceed one block's shared memory (at most " +
                std::to_string(kMaxSmem / smem_render(1)) + ")");
  if (rc->npixel > kRenderMaxPixels) return fail(std::string(what) + ": " + std::to_string(rc->npixel) + " pixels exceed " + std::to_string(kRenderMaxPixels));
  if (rc->nlight != m->dev.nlight) return fail(std::string(what) + ": the render context has " + std::to_string(rc->nlight) + " lights, the model " + std::to_string(m->dev.nlight));
  if (rc->nb_cam_fovy < 1 || rc->nb_cam_intrinsic < 1 || rc->nb_light_attenuation < 1 || rc->nb_light_cutoff < 1 || rc->nb_light_exponent < 1 ||
      rc->nb_light_ambient < 1 || rc->nb_light_diffuse < 1 || rc->nb_light_specular < 1 || rc->nb_mat_specular < 1 || rc->nb_mat_shininess < 1 ||
      rc->nb_mat_emission < 1)
    return fail(std::string(what) + ": per-world field counts must be >= 1");
  (void)d;
  return 0;
}
int mjb_refit_bvh(const mjbModel* m, mjbData* d, const mjbRender* rc, void* stream) {
  MJB_ENTER();
  if (check_render(m, d, rc, "mjb_refit_bvh")) return -1;
  MJB_LAUNCH(launch_refit_bvh(m->dev, d->dev, *rc, s));
  return 0;
}
int mjb_render(const mjbModel* m, mjbData* d, const mjbRender* rc, void* stream) {
  MJB_ENTER();
  if (check_render(m, d, rc, "mjb_render")) return -1;
  if (rc->npixel > 0 && (!rc->cam_id || !rc->cam_res || !rc->pix_adr || !rc->rgb_adr || !rc->depth_adr || !rc->seg_adr))
    return fail("mjb_render: null camera table");
  MJB_LAUNCH(launch_render(m->dev, d->dev, *rc, m->dev.nmesh > 0, s));
  return 0;
}
int mjb_render_rays(const mjbRender* rc, float* ray, void* stream) {
  g_launches = 0;
  if (!rc || !ray) return fail("mjb_render_rays: null argument");
  if (rc->npixel < 0 || rc->npixel > kRenderMaxPixels) return fail("mjb_render_rays: pixel count out of range: " + std::to_string(rc->npixel));
  if (rc->npixel > 0 && (!rc->cam_id || !rc->cam_res || !rc->pix_adr || !rc->cam_projection || !rc->cam_fovy || !rc->cam_sensorsize || !rc->cam_intrinsic))
    return fail("mjb_render_rays: null camera table");
  MJB_LAUNCH(launch_render_rays(*rc, ray, (cudaStream_t)stream));
  return 0;
}
// The k_energy parts of the position-stage sensors (sensor.py:845-849): the terms the energy sensors read, and the sensors themselves
// The sensors of `stages` (1 pos, 2 vel, 4 acc) for dd's world range: k_sensor (with the collision sensors for the position stage), then
// for the position stage the rangefinders (sensor.py:815-843), and for the acceleration stage the <contact> sensors (sensor.py:2605-2658),
// which read the solver's efc_force.  A model without rangefinders or contact sensors launches what it launched before they existed.
static cudaError_t sensors(const mjbModel* m, const mjbData* d, const DataDev& dd, int stages, cudaStream_t s) {
  cudaError_t e;
  if (mesh_large(m) && m->sc.nsensorcollision > 0) {  // the collision sensors run the CCD_MESH = 2 build, after k_sensor as launch_sensor orders them
    SensorCollisionDev none = m->sc;
    none.nsensorcollision = 0;
    e = launch_sensor(m->dev, dd, stages, s, none);
    if (e == cudaSuccess && m->dev.nsensor > 0 && (stages & 1) && !(m->dev.disableflags & DSBL_SENSOR)) e = launch_sensor_collision_large(m->dev, dd, m->sc, mesh_clip(m, d), s);
  } else {
    e = launch_sensor(m->dev, dd, stages, s, m->sc);
  }
  if (e == cudaSuccess && m->rf.nrangefinder > 0 && (stages & 1) && !(m->dev.disableflags & DSBL_SENSOR)) e = launch_sensor_rangefinder(m->dev, dd, m->rf, s);
  if (e != cudaSuccess || m->dev.nsensor == 0 || !(stages & 4) || m->scon.nsensorcontact == 0 || (m->dev.disableflags & DSBL_SENSOR)) return e;
  return launch_sensor_contact(m->dev, dd, m->scon, s);
}

static int energy_sensor_parts(const mjbModel* m) {
  if (m->en.nsensor_energy == 0 || (m->dev.disableflags & DSBL_SENSOR)) return 0;
  return ENERGY_SENSOR | (m->en.sensor_e_potential ? ENERGY_POT : 0) | (m->en.sensor_e_kinetic ? ENERGY_KIN : 0);
}
// The k_energy parts of forward (forward.py:1327-1356): with ENBL_ENERGY both terms, and the energy sensors unless DSBL_SENSOR is set (the
// reference then leaves Data.energy stale; here it is computed); without it the sensors' terms, after which Data.energy is zeroed as the
// reference does.  0 (no launch, Data.energy untouched) for a model with the flag off and no energy sensor.
static int energy_forward_parts(const mjbModel* m) {
  const int sens = energy_sensor_parts(m);
  if (m->dev.enableflags & ENBL_ENERGY) return ENERGY_POT | ENERGY_KIN | sens;
  return m->en.nsensor_energy > 0 ? sens | ENERGY_ZERO : 0;
}

int mjb_sensor_pos(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(sensors(m, d, d->dev, 1, s));
  MJB_LAUNCH(launch_energy(m->dev, d->dev, energy(m, d), energy_sensor_parts(m), s));
  MJB_LAUNCH(history_sensor(m, d, d->dev, 1, s));
  return 0;
}
int mjb_energy_pos(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_energy(m->dev, d->dev, energy(m, d), ENERGY_POT, s)); return 0; }
int mjb_energy_vel(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_energy(m->dev, d->dev, energy(m, d), ENERGY_KIN, s)); return 0; }
int mjb_sensor_vel(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(sensors(m, d, d->dev, 2, s));
  MJB_LAUNCH(history_sensor(m, d, d->dev, 2, s));
  return 0;
}
int mjb_sensor_acc(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(sensors(m, d, d->dev, 4, s));
  MJB_LAUNCH(history_sensor(m, d, d->dev, 4, s));
  return 0;
}
int mjb_solve(const mjbModel* m, mjbData* d, void* stream) { MJB_ENTER(); MJB_LAUNCH(launch_solver(m->dev, d->dev, s)); return 0; }
int mjb_euler(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(history_ctrl_insert(m, d, d->dev, s));
  MJB_LAUNCH(launch_integrate(m->dev, d->dev, INT_EULER, s, fluid(m, d)));
  return 0;
}

// which stages a pipeline call runs
enum { RUN_POSITION = 1, RUN_VELOCITY = 2, RUN_SOLVER = 4, RUN_EULER = 8, RUN_INVERSE = 16 };

// inverse.py:79-119 discrete_acc: whether the given qacc is converted from discrete time (Euler without eulerdamp=disable, implicitfast)
static bool inverse_discrete(const ModelDev& m) {
  if (!(m.enableflags & ENBL_INVDISCRETE)) return false;
  return m.integrator == INT_IMPLICITFAST || (m.integrator == INT_EULER && !(m.disableflags & DSBL_EULERDAMP));
}

// The kernels of the stages in `what` for dd's world range.  With `marks` (six events), the end of each stage group is recorded
// in the order of forward.KERNEL_NAMES: position, collision, constraint (with the CSR view), velocity, solver (with the sensors),
// integrate (every integrator kernel).
static int chain(const mjbModel* m, const mjbData* d, const DataDev& dd, int what, cudaStream_t s, cudaEvent_t* marks = nullptr) {
#define MJB_MARK(i) do { if (marks && check(cudaEventRecord(marks[i], s), "cudaEventRecord")) return -1; } while (0)
  if (what & RUN_POSITION) {
    // forward.py:635-677 with factorize=False: kinematics, com_pos, camlight, crb, collision, make_constraint, transmission
    MJB_LAUNCH(launch_position(m->dev, dd, STG_KINEMATICS | STG_COM_POS | STG_CAMLIGHT | STG_CRB | STG_TRANSMISSION, s));
    MJB_MARK(0);
    MJB_LAUNCH(collision(m, d, dd, s));
    MJB_MARK(1);
    MJB_LAUNCH(launch_constraint(m->dev, dd, s));
    if (dd.njmax_nnz > 0) MJB_LAUNCH(launch_efc_csr(m->dev, dd, s));  // sparse models: the reference's CSR arrays next to the dense rows
    MJB_MARK(2);
  }
  if (what & RUN_VELOCITY) {
    DataDev da;
    if (actuation_data(m, d, dd, s, &da)) return -1;
    MJB_LAUNCH(launch_velocity(m->dev, da, STG_VELOCITY | STG_ACTUATION | STG_ACCELERATION, s, fluid(m, d)));
    MJB_MARK(3);
  }
  if (what & RUN_SOLVER) {
    MJB_LAUNCH(launch_solver(m->dev, dd, s));
    // sensors of all three stages in one launch after the solver (forward.py:1350-1365 interleaves them; their inputs are final by now)
    if (m->dev.nsensor > 0) MJB_LAUNCH(sensors(m, d, dd, 7, s));
    // energy after the sensors (the reference's energy_pos / energy_vel, forward.py:1327-1356): its inputs are final since fwd_velocity
    MJB_LAUNCH(launch_energy(m->dev, dd, energy(m, d), energy_forward_parts(m), s));
    MJB_LAUNCH(history_sensor(m, d, dd, 7, s));  // after every kernel that writes sensordata
    MJB_MARK(4);
  }
  if (what & RUN_INVERSE) {
    // inverse dynamics at the given qacc, then the sensors of all three stages; with a discrete-time qacc they read the continuous
    // one k_inverse wrote to the scratch, and d.qacc itself is never written
    const bool disc = inverse_discrete(m->dev);
    MJB_LAUNCH(launch_inverse(m->dev, dd, d->qfrc_inverse, d->inv_qacc, disc, s, fluid(m, d)));
    if (m->dev.nsensor > 0) {
      DataDev ds = dd;
      if (disc) ds.qacc = d->inv_qacc;
      MJB_LAUNCH(sensors(m, d, ds, 7, s));
    }
    MJB_LAUNCH(launch_energy(m->dev, dd, energy(m, d), energy_sensor_parts(m), s));  // inverse computes energy only for its sensors
    MJB_LAUNCH(history_sensor(m, d, dd, 7, s));
  }
  if (what & RUN_EULER) {
    if (m->dev.integrator == INT_IMPLICIT && smem_implicit(m->dev) > kMaxSmem) return fail("implicit integrator: the velocity-derivative scratch (18 x nbody x 32 floats) exceeds one block's shared memory");
    MJB_LAUNCH(history_ctrl_insert(m, d, dd, s));
    MJB_LAUNCH(launch_integrate(m->dev, dd, -1, s, fluid(m, d)));
    MJB_MARK(5);
  }
#undef MJB_MARK
  return 0;
}

int mjb_implicit(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  if (m->dev.integrator != INT_IMPLICIT && m->dev.integrator != INT_IMPLICITFAST) return fail("mjb_implicit: the model's integrator is Euler / RK4 (the factor-and-solve scratch is sized by the integrator the model was created with)");
  return chain(m, d, d->dev, RUN_EULER, s);
}

static int pipeline(const mjbModel* m, mjbData* d, int what, cudaStream_t s) {
  if (what & RUN_POSITION) MJB_LAUNCH(reset_contact_counters(d->dev, s));
  if (d->nsplit < 2) return chain(m, d, d->dev, what, s);
  // fork: both halves wait for everything queued on the caller's stream, run their own kernel chain, and are joined back
  if (check(cudaEventRecord(d->ev_fork, s), "cudaEventRecord")) return -1;
  const int part = (d->dev.nworld + d->nsplit - 1) / d->nsplit;
  for (int h = 0; h < d->nsplit; h++) {
    DataDev dd = d->dev;
    dd.w0 = h * part;
    dd.wn = min(part, d->dev.nworld - dd.w0);
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
int mjb_inverse(const mjbModel* m, mjbData* d, void* stream) {
  MJB_ENTER();
  if ((m->dev.enableflags & ENBL_INVDISCRETE) && (m->dev.integrator == INT_RK4 || m->dev.integrator == INT_IMPLICIT))
    return fail("mjb_inverse: discrete inverse dynamics (ENBL_INVDISCRETE) is not supported for the RK4 and implicit integrators");
  return pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_INVERSE, s);
}
// forward.py:523-555 rungekutta4, called after forward(): three more forward() evaluations with the state bookkeeping in between
static int rk4_after_forward(const mjbModel* m, mjbData* d, cudaStream_t s) {
  if (!d->rk) return fail("Runge-Kutta scratch missing: data was finalized against a model whose integrator is not RK4");
  for (int stage = 0; stage < 4; stage++) {
    if (stage > 0 && pipeline(m, d, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER, s)) return -1;
    if (stage == 3) MJB_LAUNCH(history_ctrl_insert(m, d, d->dev, s));  // once, before the last stage advances d.time
    MJB_LAUNCH(launch_rk_stage(m->dev, d->dev, d->rk, stage, s));
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
  MJB_ENTER();
  // the step's kernel chain over all worlds on the caller's stream, between event ev[0] and the six stage-group events
  cudaEvent_t ev[7];
  int n = 0, rc = 0;
  while (n < 7 && !(rc = check(cudaEventCreate(&ev[n]), "cudaEventCreate"))) n++;
  if (!rc) rc = check(reset_contact_counters(d->dev, s), "reset_contact_counters");
  if (!rc) rc = check(cudaEventRecord(ev[0], s), "cudaEventRecord");
  if (!rc) rc = chain(m, d, d->dev, RUN_POSITION | RUN_VELOCITY | RUN_SOLVER | RUN_EULER, s, ev + 1);
  if (!rc) rc = check(cudaEventSynchronize(ev[6]), "cudaEventSynchronize");
  for (int i = 0; i < 6 && !rc; i++) rc = check(cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]), "cudaEventElapsedTime");
  for (int i = 0; i < n; i++) cudaEventDestroy(ev[i]);
  return rc;
}
const char* mjb_collision_kernel(const mjbModel* m) {
  if (!m || !m->finalized) { fail("model not finalized"); return nullptr; }
  if (m->dev.nmesh == 0) return "k_collision";
  return mesh_large(m) ? "k_collision_mesh_large" : "k_collision_mesh";
}
int mjb_team_residency(const mjbModel* m, const mjbData* d, int* position_worlds, int* velocity_worlds, int* shapes) {
  if (!m || !d || !m->finalized || !d->finalized) return fail("model/data not finalized");
  if (!position_worlds || !velocity_worlds) return fail("mjb_team_residency: null output");
  int local[8];
  int* sh = shapes ? shapes : local;
  if (check(resident_worlds_position(m->dev, d->dev, position_worlds, sh), "resident_worlds_position")) return -1;
  if (check(resident_worlds_velocity(m->dev, d->dev, velocity_worlds, sh + 4, fluid(m, d)), "resident_worlds_velocity")) return -1;
  return 0;
}
int mjb_set_const(const mjbModel* m, mjbData* d, int parts, int restore, void* stream) {
  MJB_ENTER();
  if (parts < 1 || parts > (MJB_SET_CONST_FIXED | MJB_SET_CONST_0 | MJB_SET_CONST_SPRING)) return fail("mjb_set_const: parts must be a non-empty combination of MJB_SET_CONST_FIXED / _0 / _SPRING, got " + std::to_string(parts));
  if (restore != 0 && restore != 1) return fail("mjb_set_const: restore must be 0 or 1");
  const ModelDev& md = m->dev;
  const int nworld = d->dev.nworld;
  const bool fixed = parts & MJB_SET_CONST_FIXED, zero = parts & MJB_SET_CONST_0, spring = (parts & MJB_SET_CONST_SPRING) && md.ntendon > 0;
  if (zero && (!m->setc.actuator_acc0 || !m->setc.meaninertia)) return fail("mjb_set_const: model array not set: actuator_acc0 / meaninertia");
  // the worlds each part stores: a derived field with nb entries takes worlds [0, nb)
  int w_zero = 1, w_spring = md.nb_tendon_lengthspring;
  struct { const char* name; int nb; } out[] = {
    {"body_subtreemass", fixed ? md.nb_body_subtreemass : 1}, {"tendon_lengthspring", spring ? md.nb_tendon_lengthspring : 1},
    {"tendon_length0", md.nb_tendon_length0}, {"eq_data", md.nb_eq_data}, {"dof_invweight0", md.nb_dof_invweight0}, {"body_invweight0", md.nb_body_invweight0},
    {"tendon_invweight0", md.nb_tendon_invweight0}, {"cam_pos0", md.nb_cam_pos0}, {"cam_poscom0", md.nb_cam_poscom0}, {"cam_mat0", md.nb_cam_mat0},
    {"light_pos0", md.nb_light_pos0}, {"light_poscom0", md.nb_light_poscom0}, {"light_dir0", md.nb_light_dir0}, {"actuator_acc0", m->setc.nb_actuator_acc0},
    {"actuator_biasprm", md.nb_actuator_biasprm}};
  for (size_t i = 0; i < sizeof(out) / sizeof(out[0]); i++) {
    const int nb = (i < 2 || zero) ? out[i].nb : 1;
    if (nb > nworld) return fail(std::string("mjb_set_const: Model.") + out[i].name + " has " + std::to_string(nb) + " entries, more than the Data's " + std::to_string(nworld) + " worlds");
    if (i >= 2) w_zero = std::max(w_zero, nb);
  }
  if (zero && smem_set_const(md) > kMaxSmem) {
    char buf[200];
    snprintf(buf, sizeof buf, "mjb_set_const: the factor and 64 right-hand-side columns of one world need %zu B of shared memory (> %zu)", smem_set_const(md), kMaxSmem);
    return fail(buf);
  }
  SetConstDev c = m->setc;
  c.qpos_save = d->qpos_save;
  if (fixed) MJB_LAUNCH(launch_set_const_fixed(md, md.nb_body_subtreemass, nworld, s));
  const int nw = std::max(zero ? w_zero : 0, spring ? w_spring : 0);  // worlds that run the position stages at qpos0 / qpos_spring
  if (nw == 0) return 0;
  DataDev dd = d->dev;
  dd.w0 = 0;
  dd.wn = nw;
  if (zero) {
    // set_const.py:656-668: the position stages and the factor of M at qpos0, then every right-hand side of a world in one warp
    MJB_LAUNCH(launch_set_const_qpos(md, dd, c, QPOS_SAVE_LOAD0, nw, s));
    MJB_LAUNCH(launch_position(md, dd, STG_KINEMATICS | STG_COM_POS | STG_CAMLIGHT | STG_CRB | STG_TRANSMISSION, s));
    MJB_LAUNCH(launch_velocity(md, dd, STG_FACTOR_ONLY, s, fluid(m, d)));
    MJB_LAUNCH(launch_set_const_0(md, dd, c, w_zero, s));
  }
  if (spring) {
    // set_const.py:856-870: kinematics, com_pos, tendon and transmission at qpos_spring
    MJB_LAUNCH(launch_set_const_qpos(md, dd, c, zero ? QPOS_LOADSPRING : QPOS_SAVE_LOADSPRING, nw, s));
    MJB_LAUNCH(launch_position(md, dd, STG_KINEMATICS | STG_COM_POS | STG_TRANSMISSION, s));
    MJB_LAUNCH(launch_set_const_spring(md, dd, w_spring, s));
  }
  MJB_LAUNCH(launch_set_const_qpos(md, dd, c, QPOS_RESTORE, nw, s));
  if (restore) {
    // set_const.py:835-844, 874-878, 940-949: the position stages and the factor of M at the restored qpos, for every world
    MJB_LAUNCH(launch_position(md, d->dev, STG_KINEMATICS | STG_COM_POS | STG_CAMLIGHT | STG_CRB | STG_TRANSMISSION, s));
    MJB_LAUNCH(launch_velocity(md, d->dev, STG_FACTOR_ONLY, s, fluid(m, d)));
  }
  return 0;
}

int mjb_set_length_range(const mjbModel* m, mjbData* d, int index, void* stream) {
  MJB_ENTER();
  const ModelDev& md = m->dev;
  if (index < -1 || index >= md.nu) return fail("mjb_set_length_range: index must be -1 or an actuator id in [0, " + std::to_string(md.nu) + "), got " + std::to_string(index));
  const int nb = md.nb_actuator_lengthrange, nworld = d->dev.nworld;
  if (nb > nworld) return fail("mjb_set_length_range: Model.actuator_lengthrange has " + std::to_string(nb) + " entries, more than the Data's " + std::to_string(nworld) + " worlds");
  MJB_LAUNCH(launch_set_length_range(md, nb, nworld, s));
  return 0;
}

// history.py:634-925 read_ctrl / read_sensor / init_ctrl_history / init_sensor_history, every world
static int history_check(const mjbModel* m, int sensor, int id, bool need_buffer) {
  const int count = sensor ? m->dev.nsensor : m->dev.nu;
  const char* what = sensor ? "sensor" : "actuator";
  if (id < 0 || id >= count) return fail(std::string(what) + " id " + std::to_string(id) + " out of range [0, " + std::to_string(count) + ")");
  if (need_buffer) {
    int n = 0;
    if (check(cudaMemcpy(&n, (sensor ? m->hist.sensor_history : m->hist.actuator_history) + 2 * id, sizeof(int), cudaMemcpyDeviceToHost), "cudaMemcpy(history)")) return -1;
    if (n <= 0) return fail(std::string(what) + " " + std::to_string(id) + " has no history buffer (nsample = 0)");
  }
  return 0;
}
static int history_read(const mjbModel* m, mjbData* d, int sensor, int id, const float* time, int interp, float* result, void* stream) {
  MJB_ENTER();
  if (!time || !result) return fail("null array");
  if (interp < -1 || interp > 2) return fail("interp must be -1 (the model's), 0 (zoh), 1 (linear) or 2 (cubic), got " + std::to_string(interp));
  if (history_check(m, sensor, id, false)) return -1;
  MJB_LAUNCH(launch_history_read(m->dev, d->dev, history(m, d), sensor, id, time, interp, result, s));
  return 0;
}
static int history_init(const mjbModel* m, mjbData* d, int sensor, int id, const float* times, const float* values, const float* phase, void* stream) {
  MJB_ENTER();
  if (!values || (sensor && !phase)) return fail("null array");
  if (history_check(m, sensor, id, true)) return -1;
  MJB_LAUNCH(launch_history_init(m->dev, d->dev, history(m, d), sensor, id, times, values, phase, s));
  return 0;
}
int mjb_read_ctrl(const mjbModel* m, mjbData* d, int ctrlid, const float* time, int interp, float* result, void* stream) { return history_read(m, d, 0, ctrlid, time, interp, result, stream); }
int mjb_read_sensor(const mjbModel* m, mjbData* d, int sensorid, const float* time, int interp, float* result, void* stream) { return history_read(m, d, 1, sensorid, time, interp, result, stream); }
int mjb_init_ctrl_history(const mjbModel* m, mjbData* d, int ctrlid, const float* times, const float* values, void* stream) {
  return history_init(m, d, 0, ctrlid, times, values, nullptr, stream);
}
int mjb_init_sensor_history(const mjbModel* m, mjbData* d, int sensorid, const float* times, const float* values, const float* phase, void* stream) {
  return history_init(m, d, 1, sensorid, times, values, phase, stream);
}

int mjb_ctrl_noise(const mjbModel* m, mjbData* d, const float* ctrl_center, int step, float noise_std, float noise_rate, void* stream) {
  MJB_ENTER();
  MJB_LAUNCH(launch_ctrl_noise(m->dev, d->dev, ctrl_center, step, noise_std, noise_rate, s));
  return 0;
}

}  // extern "C"
