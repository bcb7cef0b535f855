// mjb_types.cuh -- device-side Model / Data descriptors (plain structs of pointers + sizes).
// Field names follow the reference's Model/Data dataclasses (/root/reference/mujoco_warp/_src/types.py:982,2075).
// The X-macro lists below are the single source of truth for the by-name C-ABI setters in capi.cu.
#pragma once
#include <cuda_runtime.h>

// ---------------------------------------------------------------- Model
#define MJB_MODEL_INTS(X) \
  X(nq) X(nv) X(nu) X(nbody) X(njnt) X(ngeom) X(nsite) X(ncam) X(nlight) X(nC) X(ntree) X(nJmom) X(nlevel) \
  X(nxn_npair) X(nlimit) X(nfricdof) X(nmaxpyramid) X(integrator) X(cone) X(solver) X(iterations) \
  X(ls_iterations) X(disableflags) X(enableflags) X(broadphase) X(broadphase_filter) X(qld_total) X(maxtree) X(has_multicontact_geom) X(neq) X(nlimit_ball) X(has_gravcomp) X(nmocap) X(npair) X(has_convex_pair) X(ccd_iterations) X(epa_iterations) X(nsensor) X(nsensordata) X(sensor_subtree_vel) X(sensor_rne_postconstraint) X(nmesh) X(na) X(ntendon) X(nJten) X(ntenfric) X(nwrap) X(nmat) X(nmeshface)
#define MJB_MODEL_FLOATS(X) \
  X(timestep) X(tolerance) X(ls_tolerance) X(impratio_invsqrt) X(meaninertia) X(gravity_x) X(gravity_y) X(gravity_z) X(ccd_tolerance)
#define MJB_MODEL_IARRS(X) \
  X(body_parentid) X(body_rootid) X(body_weldid) X(body_mocapid) X(body_jntnum) X(body_jntadr) X(body_dofnum) X(body_dofadr) \
  X(body_childadr) X(body_childid) X(level_adr) X(level_body) \
  X(jnt_type) X(jnt_qposadr) X(jnt_dofadr) X(jnt_bodyid) X(jnt_actfrclimited) X(jnt_actgravcomp) X(jnt_limited_adr) \
  X(dof_bodyid) X(dof_jntid) X(dof_parentid) X(dof_fricloss_adr) X(M_rownnz) X(M_rowadr) X(M_colind) X(M_entry_row) X(mulm_rowadr) X(mulm_col) X(mulm_madr) \
  X(tree_dofadr) X(tree_dofnum) X(tree_qLDadr) \
  X(geom_type) X(geom_condim) X(geom_bodyid) X(geom_priority) \
  X(actuator_trnid) X(actuator_gaintype) X(actuator_biastype) X(actuator_ctrllimited) X(actuator_forcelimited) \
  X(actuator_dyntype) X(actuator_actadr) X(actuator_actnum) X(actuator_actlimited) X(actuator_actearly) X(actuator_trntype) \
  X(ten_J_rownnz) X(ten_J_rowadr) X(ten_J_colind) X(tendon_adr) X(tendon_num) X(wrap_objid) X(tendon_limited) X(tendon_actfrclimited) \
  X(moment_rownnz0) X(moment_rowadr0) X(moment_colind0) X(dofact_adr) X(dofact_act) X(dofact_mom) \
  X(cam_mode) X(cam_bodyid) X(cam_targetbodyid) X(light_mode) X(light_bodyid) X(light_targetbodyid) X(site_bodyid) \
  X(nxn_geom_pair) X(nxn_pairid) X(body_isdofancestor) X(eq_type) X(eq_obj1id) X(eq_obj2id) X(jnt_limited_ball_adr) X(pair_dim) \
  X(sensor_type) X(sensor_datatype) X(sensor_needstage) X(sensor_objtype) X(sensor_objid) X(sensor_reftype) X(sensor_refid) X(sensor_dim) X(sensor_adr) X(site_type) \
  X(geom_dataid) X(mesh_vertadr) X(mesh_vertnum) X(mesh_graphadr) X(mesh_graph) X(mesh_polynum) X(mesh_polyadr) X(mesh_polyvertadr) X(mesh_polyvertnum) \
  X(mesh_polyvert) X(mesh_polymapadr) X(mesh_polymapnum) X(mesh_polymap) X(geom_group) X(geom_matid) X(mesh_faceadr) X(mesh_face) X(jnt_limited)
#define MJB_MODEL_FARRS(X) \
  X(qpos0) X(qpos_spring) X(body_pos) X(body_quat) X(body_ipos) X(body_iquat) X(body_mass) X(body_subtreemass) \
  X(body_inertia) X(body_invweight0) X(body_gravcomp) X(jnt_pos) X(jnt_axis) X(jnt_stiffness) X(jnt_range) X(jnt_margin) X(jnt_solref) \
  X(jnt_solimp) X(jnt_actfrcrange) X(dof_armature) X(dof_damping) X(dof_invweight0) X(dof_frictionloss) X(dof_solref) \
  X(dof_solimp) X(geom_size) X(geom_aabb) X(geom_rbound) X(geom_pos) X(geom_quat) X(geom_friction) X(geom_margin) \
  X(geom_gap) X(geom_solmix) X(geom_solref) X(geom_solimp) X(actuator_gear) X(actuator_gainprm) X(actuator_biasprm) \
  X(actuator_ctrlrange) X(actuator_forcerange) X(cam_pos) X(cam_quat) X(cam_poscom0) X(cam_pos0) X(cam_mat0) \
  X(light_pos) X(light_dir) X(light_poscom0) X(light_pos0) X(light_dir0) X(site_pos) X(site_quat) \
  X(eq_solref) X(eq_solimp) X(eq_data) X(pair_friction) X(pair_solref) X(pair_solreffriction) X(pair_solimp) X(pair_margin) X(pair_gap) \
  X(sensor_cutoff) X(site_size) X(mesh_vert) X(mesh_polynormal) X(actuator_dynprm) X(actuator_actrange) \
  X(wrap_prm) X(ten_J0) X(tendon_range) X(tendon_margin) X(tendon_stiffness) X(tendon_damping) X(tendon_frictionloss) X(tendon_lengthspring) \
  X(tendon_length0) X(tendon_invweight0) X(tendon_solref_lim) X(tendon_solimp_lim) X(tendon_solref_fri) X(tendon_solimp_fri) X(tendon_actfrcrange) \
  X(geom_rgba) X(mat_rgba) X(actuator_acc0) X(actuator_lengthrange)
// opt.magnetic (nb, 3), cam_fovy (nb, ncam), cam_intrinsic (nb, ncam, 4), cam_sensorsize (ncam, 2): batched like MJB_MODEL_FARRS
#define MJB_MODEL_SENSOR_FARRS(X) X(magnetic) X(cam_fovy) X(cam_intrinsic) X(cam_sensorsize)

struct ModelDev {
#define X(n) int n;
  MJB_MODEL_INTS(X)
#undef X
#define X(n) float n;
  MJB_MODEL_FLOATS(X)
#undef X
#define X(n) const int* __restrict__ n;
  MJB_MODEL_IARRS(X)
#undef X
#define X(n) const float* __restrict__ n;
  MJB_MODEL_FARRS(X)
#undef X
  // per-world (batched) float fields, the reference's `*` leading dimension (types.py:822-833, io.py:259-282): world w reads entry
  // w % nb of a field with nb > 1 entries of bs floats each.  batched = any field has nb > 1 (selects the BAT kernel instantiations).
  int batched;
#define X(n) int nb_##n, bs_##n;
  MJB_MODEL_FARRS(X)
#undef X
  // fields only the magnetometer / camprojection / insidesite / tendon sensors read (k_sensor's EXTRA build): appended after every other
  // field, so that the parameter offsets of every other kernel stay where they were
  int sensor_extra;                                  // the model has a sensor of one of those types (selects k_sensor<BAT, true>)
  const int* __restrict__ cam_resolution;            // (ncam, 2)
#define X(n) const float* __restrict__ n; int nb_##n, bs_##n;
  MJB_MODEL_SENSOR_FARRS(X)
#undef X
};

#ifdef __CUDACC__
// The model as world w sees it: every batched float field already offset to the world's entry.  Unused fields cost nothing (the
// copy is scalar-replaced); with one world per warp the offsets stay in uniform registers.
__device__ __forceinline__ ModelDev world_model(const ModelDev& m, int w, int nworld) {
  ModelDev r = m;
#define X(n) if (m.nb_##n > 1) r.n = m.n + (size_t)(m.nb_##n == nworld ? w : w % m.nb_##n) * (size_t)m.bs_##n;
  MJB_MODEL_FARRS(X)
  MJB_MODEL_SENSOR_FARRS(X)
#undef X
  return r;
}
// Inside a kernel template with `bool BAT` whose Model parameter is `mp`: defines `m`, the model of world `w`.
#define MJB_WORLD_MODEL(w)                                         \
  ModelDev m_world_;                                               \
  if (BAT) m_world_ = world_model(mp, (w), d.nworld);              \
  const ModelDev& m = BAT ? m_world_ : mp;
#endif

// ---------------------------------------------------------------- Data
#define MJB_DATA_FARRS(X) \
  X(time) X(qpos) X(qvel) X(ctrl) X(qacc_warmstart) X(qfrc_applied) X(xfrc_applied) X(qacc) \
  X(xpos) X(xquat) X(xmat) X(xipos) X(ximat) X(xanchor) X(xaxis) X(geom_xpos) X(geom_xmat) X(site_xpos) X(site_xmat) \
  X(cam_xpos) X(cam_xmat) X(light_xpos) X(light_xdir) X(subtree_com) X(cdof) X(cinert) X(crb) X(M) X(qLD) \
  X(actuator_length) X(actuator_moment) X(actuator_velocity) X(cvel) X(cdof_dot) X(qfrc_bias) X(qfrc_spring) \
  X(qfrc_damper) X(qfrc_gravcomp) X(qfrc_passive) X(actuator_force) X(qfrc_actuator) X(qfrc_smooth) X(qacc_smooth) \
  X(qfrc_constraint) X(cacc) X(cfrc_int) \
  X(efc_J) X(efc_pos) X(efc_margin) X(efc_D) X(efc_vel) X(efc_aref) X(efc_frictionloss) X(efc_force) X(efc_Ma) \
  X(contact_dist) X(contact_pos) X(contact_frame) X(contact_includemargin) X(contact_friction) X(contact_solref) \
  X(contact_solreffriction) X(contact_solimp) X(mocap_pos) X(mocap_quat) X(sensordata) X(subtree_linvel) X(subtree_angmom) X(cfrc_ext) X(efc_Jsp) X(act) X(act_dot) X(ten_length) X(ten_J) X(ten_velocity) X(qLU)
#define MJB_DATA_IARRS(X) \
  X(ne) X(nf) X(nl) X(nefc) X(nacon) X(ncollision) X(solver_niter) X(overflow) X(efc_type) X(efc_id) X(efc_state) \
  X(moment_rownnz) X(moment_rowadr) X(moment_colind) X(contact_dim) X(contact_geom) X(contact_efc_address) \
  X(contact_worldid) X(contact_type) X(contact_geomcollisionid) X(eq_active) X(efc_J_rownnz) X(efc_J_rowadr) X(efc_J_colind)

struct DataDev {
  int nworld, nconmax, naconmax, njmax, njmax_pad, nv_pad;
  int w0, wn;  // world range [w0, w0 + wn) processed by one launch (the step is pipelined over two world halves)
  int njmax_nnz;  // capacity of the CSR view of efc.J (0: dense model, no CSR view)
#define X(n) float* __restrict__ n;
  MJB_DATA_FARRS(X)
#undef X
#define X(n) int* __restrict__ n;
  MJB_DATA_IARRS(X)
#undef X
  // internal scratch (allocated by mjb_data_finalize; not part of the reference's Data)
  int* world_conadr;  // (nworld) first contact-pool slot of each world's contiguous block
  int* world_ncon;    // (nworld) number of contacts the world wrote this step
  float* imp_qacc;    // (nworld, nv) acceleration solved by the fully implicit integrator (k_implicit.cu), consumed by the advance kernel
};

// ---------------------------------------------------------------- fluid forces (mjb_fluid.cuh)
// Model and Data fields of fluid forces, passed as one extra argument to the fluid instances of k_velocity, k_euler and k_inverse only:
// adding them to ModelDev / DataDev would move the kernel parameters of every other kernel.  density / viscosity / wind are model
// constants (the reference indexes them per world).
#define MJB_FLUID_INTS(X) X(has_fluid)
#define MJB_FLUID_FLOATS(X) X(density) X(viscosity) X(wind_x) X(wind_y) X(wind_z)
#define MJB_FLUID_IARRS(X) X(body_fluid) X(body_geomadr) X(body_geomnum)
#define MJB_FLUID_FARRS(X) X(geom_fluid)
struct FluidDev {
  int has_fluid;                         // opt.density > 0, opt.viscosity > 0 or a non-zero opt.wind
  float density, viscosity, wind_x, wind_y, wind_z;
  const int* __restrict__ body_fluid;    // (nbody) FLUID_NONE / FLUID_ELLIPSOID / FLUID_BOX
  const int* __restrict__ body_geomadr;  // (nbody)
  const int* __restrict__ body_geomnum;  // (nbody)
  const float* __restrict__ geom_fluid;  // (ngeom, 12), MuJoCo's layout
  float* __restrict__ qfrc_fluid;        // Data.qfrc_fluid (nworld, nv)
};

// ---------------------------------------------------------------- collision sensors (k_sensor_collision.cu)
// The geom pairs of the distance / normal / fromto sensors (io.py _sensor_collision_tables), passed as one extra argument to
// k_sensor_collision only, for the same reason as FluidDev.  They stay off nxn_pairid: the contact pipeline never sees them.
#define MJB_SENSCOL_INTS(X) X(nsensorcollision) X(nsensorcollision_sensor) X(nsensorcollision_ccd) X(sensor_collision_epa_iterations)
#define MJB_SENSCOL_IARRS(X) X(sensor_collision_start_adr) X(sensor_collision_pair) X(sensor_collision_id) X(sensor_collision_adr) X(sensor_collision_flip)
struct SensorCollisionDev {
  int nsensorcollision;                                // unique geom pairs
  int nsensorcollision_sensor;                         // distance / normal / fromto sensors
  int nsensorcollision_ccd;                            // pairs that run GJK / EPA (one scratch slot each, at most 32 in use)
  int sensor_collision_epa_iterations;
  const int* __restrict__ sensor_collision_start_adr;  // (sum over sensors of n1 n2) unique-pair index of each (sensor, geom1, geom2)
  const int* __restrict__ sensor_collision_pair;       // (nsensorcollision, 4) geoms in narrowphase order, explicit <pair> id or -1,
                                                       // GJK / EPA rank among the pairs or -1
  const int* __restrict__ sensor_collision_id;         // (nsensorcollision_sensor) sensor ids
  const int* __restrict__ sensor_collision_adr;        // (nsensorcollision_sensor + 1) first start_adr entry of each sensor
  const int* __restrict__ sensor_collision_flip;       // (like start_adr) the entry's geom1 is the narrowphase's second geom
};

// ---------------------------------------------------------------- contact sensors (k_sensor_contact.cu, mjb_sensor_contact.cuh)
// The <contact> sensors' tables and Option.contact_sensor_maxmatch, passed as one extra argument to k_sensor_contact only, for the same
// reason as FluidDev.
#define MJB_SENSCON_INTS(X) X(nsensorcontact) X(contact_sensor_maxmatch)
#define MJB_SENSCON_IARRS(X) X(sensor_contact_adr) X(sensor_intprm)
struct SensorContactDev {
  int nsensorcontact;                          // contact sensors
  int contact_sensor_maxmatch;                 // matches kept per sensor and world (the rest are counted, and raise OVF_CONTACT_MATCH)
  const int* __restrict__ sensor_contact_adr;  // (nsensorcontact) their sensor ids
  const int* __restrict__ sensor_intprm;       // (nsensor, 3) dataspec, reduce, num of each contact sensor; zeros for the others
};

// ---------------------------------------------------------------- rangefinders (k_sensor_rangefinder.cu)
// The rangefinder tables (reference io.py:885-887, :910), passed as one extra argument to k_sensor_rangefinder only, for the same reason
// as FluidDev.  k_sensor skips the rangefinders' slots; this kernel writes them.
#define MJB_RANGEFINDER_INTS(X) X(nrangefinder)
#define MJB_RANGEFINDER_IARRS(X) X(sensor_rangefinder_adr) X(sensor_rangefinder_bodyid)
struct RangefinderDev {
  int nrangefinder;                                   // rangefinder sensors
  const int* __restrict__ sensor_rangefinder_adr;     // (nrangefinder) their sensor ids
  const int* __restrict__ sensor_rangefinder_bodyid;  // (nrangefinder) the body of each one's site (excluded from its ray)
};

// ---------------------------------------------------------------- set_const (k_set_const.cu)
// The fields of mjb_set_const that are neither in ModelDev nor in DataDev, passed as one extra argument to its kernels only, for the
// same reason as FluidDev.  Writes to the other derived Model fields go through ModelDev's pointers and nb_* / bs_*.
struct SetConstDev {
  float* __restrict__ actuator_acc0;  // Model.actuator_acc0 (nb_actuator_acc0, nu)
  int nb_actuator_acc0;
  float* __restrict__ meaninertia;    // Model.stat.meaninertia on the device (1): world 0's value
  float* __restrict__ qpos_save;      // (nworld, nq) d.qpos while qpos0 / qpos_spring stand in for it (mjb_data_finalize allocates it)
};
enum { QPOS_SAVE_LOAD0 = 0, QPOS_SAVE_LOADSPRING = 1, QPOS_LOADSPRING = 2, QPOS_RESTORE = 3 };  // k_set_const_qpos modes

// ---------------------------------------------------------------- energy (k_energy.cu)
// Data.energy and the e_potential / e_kinetic sensors, passed as one extra argument to k_energy only, for the same reason as FluidDev.
#define MJB_ENERGY_INTS(X) X(nsensor_energy) X(sensor_e_potential) X(sensor_e_kinetic)
#define MJB_ENERGY_IARRS(X) X(sensor_energy_adr)
struct EnergyDev {
  int nsensor_energy;                         // e_potential and e_kinetic sensors
  int sensor_e_potential, sensor_e_kinetic;   // the model has a sensor of that type
  const int* __restrict__ sensor_energy_adr;  // (nsensor_energy) their sensor ids
  float* __restrict__ energy;                 // Data.energy (nworld, 2): potential, kinetic
};
// k_energy parts: the potential and kinetic terms into Data.energy, the energy sensors from them, and Data.energy zeroed afterwards
// (forward with ENBL_ENERGY off: the sensors report, Data.energy ends at zero)
enum { ENERGY_POT = 1, ENERGY_KIN = 2, ENERGY_SENSOR = 4, ENERGY_ZERO = 8 };

// ---------------------------------------------------------------- actuator and sensor delays (k_history.cu, mjb_history.cuh)
// The delay / history fields of the Model and Data.history, passed as one extra argument to the k_history kernels only, for the same
// reason as FluidDev.  Buffers are laid out as [user, cursor, times[n], values[n * dim]] at *_historyadr of each world's row.
#define MJB_HISTORY_INTS(X) X(nhistory) X(nactuator_history) X(nsensor_history)
#define MJB_HISTORY_IARRS(X) X(actuator_history) X(actuator_historyadr) X(sensor_history) X(sensor_historyadr) X(sensor_history_id)
#define MJB_HISTORY_FARRS(X) X(actuator_delay) X(sensor_delay) X(sensor_interval)
struct HistoryDev {
  int nhistory;                                 // floats of history per world
  int nactuator_history;                        // actuators with nsample > 0
  int nsensor_history;                         // sensors with nsample > 0
  const int* __restrict__ actuator_history;     // (nu, 2) nsample, interp
  const int* __restrict__ actuator_historyadr;  // (nu) buffer address or -1
  const int* __restrict__ sensor_history;       // (nsensor, 2)
  const int* __restrict__ sensor_historyadr;    // (nsensor)
  const int* __restrict__ sensor_history_id;    // (nsensor_history) the sensors with nsample > 0
  const float* __restrict__ actuator_delay;     // (nu)
  const float* __restrict__ sensor_delay;       // (nsensor)
  const float* __restrict__ sensor_interval;    // (nsensor, 2) period, phase
  float* __restrict__ history;                  // Data.history (nworld, nhistory)
  float* __restrict__ ctrl_delayed;             // (nworld, nu) the ctrl k_velocity's actuation reads (mjb_data_finalize allocates it)
};

// ---------------------------------------------------------------- mesh multi-contact scratch (k_collision_mesh_large.cu, k_sensor_collision_large.cu)
// Models whose hulls have a polygon of more than kMeshPolyCap vertices, or a vertex shared by more than kMeshDegCap polygons, run the CCD_MESH = 2
// build of the collision and collision-sensor kernels.  Its multi-contact buffers are sized from the model and live in global scratch: nslot
// slices per world, one per lane that runs GJK / EPA at once.  Passed as one extra argument to those kernels only, for the same reason as FluidDev.
constexpr int kMeshPolyCap = 32, kMeshDegCap = 16;  // the fixed buffers of the CCD_MESH = 1 build (mjb_ccd.cuh)
#define MJB_MESHCLIP_INTS(X) X(npolygonmax) X(nmeshdegmax)
struct MeshClipDev {
  int npolygonmax;              // Model.npolygonmax: most vertices in one hull polygon
  int nmeshdegmax;              // Model.nmeshdegmax: most hull polygons at one vertex
  int nslot;                    // scratch slices per world
  float* __restrict__ scratch;  // (nworld, nslot, mesh_clip_words) allocated by mjb_data_finalize for such models only
};
__host__ __device__ inline bool mesh_clip_large(int npolygonmax, int nmeshdegmax) { return npolygonmax > kMeshPolyCap || nmeshdegmax > kMeshDegCap; }
// buffer sizes: the model's, and at least a box's 4-vertex face / 3 faces at a corner
__host__ __device__ inline int mesh_clip_poly(const MeshClipDev& c) { return c.npolygonmax > 4 ? c.npolygonmax : 4; }
__host__ __device__ inline int mesh_clip_deg(const MeshClipDev& c) { return c.nmeshdegmax > 3 ? c.nmeshdegmax : 3; }
// floats of one slice: candidate normals of each geom and the edge end vertices (3 maxdeg each), the polygon ids of each geom's normals (maxdeg
// each), the two faces (3 maxpoly each) and the two clip buffers (3 x 2 maxpoly each)
__host__ __device__ inline int mesh_clip_words(int maxpoly, int maxdeg) { return 11 * maxdeg + 18 * maxpoly; }
__host__ __device__ inline int mesh_clip_words(const MeshClipDev& c) { return mesh_clip_words(mesh_clip_poly(c), mesh_clip_deg(c)); }

// ---------------------------------------------------------------- enums (MuJoCo values; see constants.py)
enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum { GEOM_PLANE = 0, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH };
enum { INT_EULER = 0, INT_RK4, INT_IMPLICIT, INT_IMPLICITFAST };
enum { CONE_PYRAMIDAL = 0, CONE_ELLIPTIC = 1 };
enum { SOL_CG = 1, SOL_NEWTON = 2 };
enum { EQ_CONNECT = 0, EQ_WELD = 1, EQ_JOINT = 2, EQ_TENDON = 3 };
enum { TRN_JOINT = 0, TRN_TENDON = 3 };
enum { OBJ_BODY = 1, OBJ_XBODY = 2, OBJ_GEOM = 5, OBJ_SITE = 6, OBJ_CAMERA = 7 };
// mjtSensor values of the sensor types carried here (MuJoCo order, as in _src/constants.py)
enum { SENS_TOUCH = 0, SENS_ACCELEROMETER = 1, SENS_VELOCIMETER = 2, SENS_GYRO = 3, SENS_FORCE = 4, SENS_TORQUE = 5, SENS_MAGNETOMETER = 6, SENS_RANGEFINDER = 7, SENS_CAMPROJECTION = 8, SENS_JOINTPOS = 9, SENS_JOINTVEL = 10, SENS_TENDONPOS = 11, SENS_TENDONVEL = 12, SENS_ACTUATORPOS = 13, SENS_ACTUATORVEL = 14,
       SENS_ACTUATORFRC = 15, SENS_JOINTACTFRC = 16, SENS_TENDONACTFRC = 17, SENS_BALLQUAT = 18, SENS_BALLANGVEL = 19, SENS_JOINTLIMITPOS = 20, SENS_JOINTLIMITVEL = 21, SENS_JOINTLIMITFRC = 22, SENS_TENDONLIMITPOS = 23,
       SENS_TENDONLIMITVEL = 24, SENS_TENDONLIMITFRC = 25, SENS_FRAMEPOS = 26, SENS_FRAMEQUAT = 27, SENS_FRAMEXAXIS = 28,
       SENS_FRAMEYAXIS = 29, SENS_FRAMEZAXIS = 30, SENS_FRAMELINVEL = 31, SENS_FRAMEANGVEL = 32, SENS_FRAMELINACC = 33, SENS_FRAMEANGACC = 34, SENS_SUBTREECOM = 35, SENS_SUBTREELINVEL = 36, SENS_SUBTREEANGMOM = 37, SENS_INSIDESITE = 38, SENS_GEOMDIST = 39, SENS_GEOMNORMAL = 40,
       SENS_GEOMFROMTO = 41, SENS_E_POTENTIAL = 43, SENS_E_KINETIC = 44, SENS_CLOCK = 45 };
enum { CNSTR_EQUALITY = 0, CNSTR_FRICTION_DOF = 1, CNSTR_FRICTION_TENDON = 2, CNSTR_LIMIT_JOINT = 3, CNSTR_LIMIT_TENDON = 4, CNSTR_CONTACT_FRICTIONLESS = 5, CNSTR_CONTACT_PYRAMIDAL = 6, CNSTR_CONTACT_ELLIPTIC = 7 };
enum { ST_SATISFIED = 0, ST_QUADRATIC = 1, ST_LINEARNEG = 2, ST_LINEARPOS = 3, ST_CONE = 4 };
enum { CAM_FIXED = 0, CAM_TRACK, CAM_TRACKCOM, CAM_TARGETBODY, CAM_TARGETBODYCOM };
enum { GAIN_FIXED = 0, GAIN_AFFINE = 1, GAIN_MUSCLE = 2 };
enum { DYN_NONE = 0, DYN_INTEGRATOR = 1, DYN_FILTER = 2, DYN_FILTEREXACT = 3, DYN_MUSCLE = 4 };
enum { BIAS_NONE = 0, BIAS_AFFINE = 1, BIAS_MUSCLE = 2 };
enum {
  DSBL_CONSTRAINT = 1 << 0, DSBL_EQUALITY = 1 << 1, DSBL_FRICTIONLOSS = 1 << 2, DSBL_LIMIT = 1 << 3, DSBL_CONTACT = 1 << 4,
  DSBL_SPRING = 1 << 5, DSBL_DAMPER = 1 << 6, DSBL_GRAVITY = 1 << 7, DSBL_CLAMPCTRL = 1 << 8, DSBL_WARMSTART = 1 << 9,
  DSBL_ACTUATION = 1 << 11, DSBL_REFSAFE = 1 << 12, DSBL_SENSOR = 1 << 13, DSBL_EULERDAMP = 1 << 15, DSBL_NATIVECCD = 1 << 17
};
enum { ENBL_ENERGY = 1 << 1, ENBL_INVDISCRETE = 1 << 3 };
enum { OVF_NEFC = 1 << 0, OVF_NJMAX_NNZ = 1 << 1, OVF_BROADPHASE = 1 << 2, OVF_NARROWPHASE = 1 << 3, OVF_CONTACT_MATCH = 1 << 6, OVF_EPA_HORIZON = 1 << 8, OVF_ITERATIONS = 1 << 9, OVF_LS_ITERATIONS = 1 << 10 };
enum { BF_PLANE = 1, BF_SPHERE = 2, BF_AABB = 4, BF_OBB = 8 };
enum { CONTACT_TYPE_CONSTRAINT = 1, CONTACT_TYPE_SENSOR = 2 };

#define MJ_MINVAL 1e-15f
#define MJ_MAXVAL 1e10f
#define MJ_MINIMP 1e-4f
#define MJ_MAXIMP 0.9999f
#define MJ_MINMU 1e-5f

// stage bits for the fused position kernel
enum { STG_KINEMATICS = 1, STG_COM_POS = 2, STG_CAMLIGHT = 4, STG_CRB = 8, STG_TRANSMISSION = 16 };
// stage bits for the fused velocity kernel
enum { STG_VELOCITY = 1, STG_ACTUATION = 2, STG_ACCELERATION = 4, STG_FACTOR_ONLY = 8,
       STG_COMVEL = 16, STG_PASSIVE = 32, STG_RNE = 64 };  // single sub-stages of fwd_velocity (smooth.com_vel, passive.passive, smooth.rne)

// launchers (one per .cu); each returns the cudaError of the launch
cudaError_t launch_position(const ModelDev& m, const DataDev& d, int stage_mask, cudaStream_t s);
cudaError_t launch_collision(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_collision_mesh(const ModelDev& m, const DataDev& d, cudaStream_t s);  // CCD_MESH build of the same kernel (k_collision_mesh.cu)
// CCD_MESH = 2 build for hulls past the fixed buffers (k_collision_mesh_large.cu); same shared memory as the CCD_MESH build
cudaError_t launch_collision_mesh_large(const ModelDev& m, const DataDev& d, const MeshClipDev& c, cudaStream_t s);
size_t smem_collision_mesh(const ModelDev& m, const DataDev& d);
cudaError_t reset_contact_counters(const DataDev& d, cudaStream_t s);
cudaError_t launch_constraint(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_efc_csr(const ModelDev& m, const DataDev& d, cudaStream_t s);  // CSR view of efc.J (sparse models)
cudaError_t launch_velocity(const ModelDev& m, const DataDev& d, int stage_mask, cudaStream_t s, const FluidDev& f);
cudaError_t launch_solve_m(const ModelDev& m, const DataDev& d, float* x, const float* y, cudaStream_t s);
cudaError_t launch_mul_m(const ModelDev& m, const DataDev& d, float* res, const float* vec, cudaStream_t s);
cudaError_t launch_solver(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_integrate(const ModelDev& m, const DataDev& d, int integrator, cudaStream_t s, const FluidDev& f);
cudaError_t launch_implicit_solve(const ModelDev& m, const DataDev& d, float* qacc_out, cudaStream_t s);  // fully implicit integrator: qLU and its solve
size_t smem_implicit(const ModelDev& m);
// the sensors of `stages` (1 pos, 2 vel, 4 acc); with the position stage also the collision sensors (k_sensor_collision.cu)
cudaError_t launch_sensor(const ModelDev& m, const DataDev& d, int stages, cudaStream_t s, const SensorCollisionDev& c);
cudaError_t launch_sensor_collision(const ModelDev& m, const DataDev& d, const SensorCollisionDev& c, cudaStream_t s);
size_t smem_sensor_collision(const SensorCollisionDev& c);
cudaError_t launch_sensor_collision_large(const ModelDev& m, const DataDev& d, const SensorCollisionDev& c, const MeshClipDev& mc, cudaStream_t s);
cudaError_t launch_contact_force(const ModelDev& m, const DataDev& d, const int* contact_ids, int n, int to_world, float* out, cudaStream_t s);
// the <contact> sensors of d's world range, after the acceleration-stage sensors (k_sensor_contact.cu)
cudaError_t launch_sensor_contact(const ModelDev& m, const DataDev& d, const SensorContactDev& c, cudaStream_t s);
size_t smem_sensor_contact(const SensorContactDev& c);
// the rangefinders of d's world range, after k_sensor's position stage (k_sensor_rangefinder.cu)
cudaError_t launch_sensor_rangefinder(const ModelDev& m, const DataDev& d, const RangefinderDev& r, cudaStream_t s);
// inverse dynamics at the given d.qacc into qfrc_inverse (nworld, nv); disc: d.qacc is a discrete-time acceleration, converted first,
// and the continuous one goes to qacc_cont (nworld, nv) (k_inverse.cu)
cudaError_t launch_inverse(const ModelDev& m, const DataDev& d, float* qfrc_inverse, float* qacc_cont, bool disc, cudaStream_t s, const FluidDev& f);
cudaError_t launch_rk_stage(const ModelDev& m, const DataDev& d, float* rk, int stage, cudaStream_t s);
// rays (nworld x nray, world-major) against every geom of every world; geomgroup: 6 ints, all -1 = no group filter (k_ray.cu)
cudaError_t launch_ray(const ModelDev& m, const DataDev& d, const float* pnt, const float* vec, int nray, int pnt_nbatch, const int* geomgroup, int flg_static,
                       const int* bodyexclude, float* dist, int* geomid, float* normal, cudaStream_t s);
// the batch renderer (k_render.cu): bounds of rc's enabled geoms in every world; one image per (world, active camera) of rc
struct mjbRender;
cudaError_t launch_refit_bvh(const ModelDev& m, const DataDev& d, const mjbRender& rc, cudaStream_t s);
cudaError_t launch_render(const ModelDev& m, const DataDev& d, const mjbRender& rc, bool has_mesh, cudaStream_t s);
cudaError_t launch_render_rays(const mjbRender& rc, float* ray, cudaStream_t s);  // the camera-frame ray table of rc's pixels
size_t smem_render(int ngeom);
constexpr int kRenderMaxPixels = 65535 * 128;  // pixels of all active cameras (tiles of 128 along the grid's y dimension)
cudaError_t launch_ctrl_noise(const ModelDev& m, const DataDev& d, const float* ctrl_center, int step, float std, float rate, cudaStream_t s);
size_t smem_position(const ModelDev& m, const DataDev& d);
size_t smem_collision(const ModelDev& m, const DataDev& d);
size_t smem_constraint(const ModelDev& m, const DataDev& d);
size_t smem_velocity(const ModelDev& m, const DataDev& d, const FluidDev& f);
// worlds per SM resident at once (occupancy API) in the launch shape k_position / k_velocity take for d's world range, and that
// shape: shape[0..3] = lanes per world, warps per block, block bytes, instance (k_velocity: 0 plain, 1 PEXT, 2 fluid; k_position: 0)
cudaError_t resident_worlds_position(const ModelDev& m, const DataDev& d, int* worlds, int* shape);
cudaError_t resident_worlds_velocity(const ModelDev& m, const DataDev& d, int* worlds, int* shape, const FluidDev& f);
size_t smem_solver(const ModelDev& m, const DataDev& d);
// set_const (k_set_const.cu): body_subtreemass of worlds [0, nw); qpos swap of worlds [0, nw); set_const_0's outputs of worlds [0, nw)
// from the position stages and factor at their qpos0; tendon_lengthspring of worlds [0, nw)
cudaError_t launch_set_const_fixed(const ModelDev& m, int nw, int nworld, cudaStream_t s);
cudaError_t launch_set_const_qpos(const ModelDev& m, const DataDev& d, const SetConstDev& c, int mode, int nw, cudaStream_t s);
cudaError_t launch_set_const_0(const ModelDev& m, const DataDev& d, const SetConstDev& c, int nw, cudaStream_t s);
cudaError_t launch_set_const_spring(const ModelDev& m, const DataDev& d, int nw, cudaStream_t s);
size_t smem_set_const(const ModelDev& m);
// set_length_range (k_set_const.cu): actuator_lengthrange of worlds [0, nw) from the joint / tendon limits and gear
cudaError_t launch_set_length_range(const ModelDev& m, int nw, int nworld, cudaStream_t s);
// energy (k_energy.cu): the ENERGY_* parts of d's world range
cudaError_t launch_energy(const ModelDev& m, const DataDev& d, const EnergyDev& e, int parts, cudaStream_t s);
size_t smem_integrate(const ModelDev& m);
// the individually callable stages that read a finished forward pass (k_body_stages.cu), each over d's world range: cacc / cfrc_int /
// cfrc_ext; subtree_linvel / subtree_angmom; the (nworld, 3, nv) Jacobians of point (nworld, 3) on body (nworld) into jacp / jacr (either
// may be null); qfrc (nworld, nv) += J^T xfrc_applied; ten_length / ten_J (no launch without tendons); out (nworld, nC) = M - dt qDeriv
cudaError_t launch_rne_postconstraint(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_subtree_vel(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_jac(const ModelDev& m, const DataDev& d, float* jacp, float* jacr, const float* point, const int* body, cudaStream_t s);
cudaError_t launch_xfrc_accumulate(const ModelDev& m, const DataDev& d, float* qfrc, cudaStream_t s);
cudaError_t launch_tendon(const ModelDev& m, const DataDev& d, cudaStream_t s);
cudaError_t launch_deriv_smooth_vel(const ModelDev& m, const DataDev& d, float* out, cudaStream_t s, const FluidDev& f);
size_t smem_deriv_smooth_vel(const ModelDev& m);
// actuator and sensor delays (k_history.cu), each over d's world range: the delayed ctrl into h.ctrl_delayed; d.ctrl inserted at
// d.time; the sensors of `stages` (1 pos, 2 vel, 4 acc) replaced by their delayed / held values, the fresh ones inserted
cudaError_t launch_history_ctrl_read(const ModelDev& m, const DataDev& d, const HistoryDev& h, cudaStream_t s);
cudaError_t launch_history_ctrl_insert(const ModelDev& m, const DataDev& d, const HistoryDev& h, cudaStream_t s);
cudaError_t launch_history_sensor(const ModelDev& m, const DataDev& d, const HistoryDev& h, int stages, cudaStream_t s);
// the public history functions, every world: one actuator's or sensor's value at time[w] - delay into result (nworld, dim); one
// buffer filled from times (n, or null: -MJ_MAXVAL stamps) and values (nworld, n * dim), its user slot set to phase[w] (sensors) or kept
cudaError_t launch_history_read(const ModelDev& m, const DataDev& d, const HistoryDev& h, int sensor, int id, const float* time, int interp, float* result, cudaStream_t s);
cudaError_t launch_history_init(const ModelDev& m, const DataDev& d, const HistoryDev& h, int sensor, int id, const float* times, const float* values, const float* phase,
                                cudaStream_t s);
