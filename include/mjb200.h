/* mjb200.h -- C ABI of the H100-native (sm_90a) batched MuJoCo physics step (libmjb200.so).
 *
 * Drop-in boundary for the step path of google-deepmind/mujoco_warp.  Every entry point replaces a
 * Python function of the reference's public API (paths relative to /root/reference/mujoco_warp/):
 *
 *   mjb_model_* / mjb_data_*   <- _src/io.py:259 put_model, :1680 make_data, :1890 put_data (device SoA binding;
 *                                 the reference binds wp.array pointers into wp.launch argument lists)
 *   mjb_step                   <- _src/forward.py:1368 step(m, d)
 *   mjb_forward                <- _src/forward.py:1341 forward(m, d)
 *   mjb_inverse                <- _src/inverse.py:148  inverse(m, d): position and velocity stages, then the constraint forces at the
 *                                                      given d.qacc and qfrc_inverse; ENBL_INVDISCRETE converts a discrete-time qacc first
 *   mjb_fwd_position           <- _src/forward.py:635  fwd_position(m, d, factorize=False)
 *   mjb_kinematics             <- _src/smooth.py:447   kinematics
 *   mjb_com_pos                <- _src/smooth.py:824   com_pos
 *   mjb_camlight               <- _src/smooth.py:984   camlight
 *   mjb_crb                    <- _src/smooth.py:1079  crb
 *   mjb_transmission           <- _src/smooth.py:2890  transmission
 *   mjb_collision              <- _src/collision_driver.py:884 collision (NXN broadphase + primitive narrowphase)
 *   mjb_make_constraint        <- _src/constraint.py:4897 make_constraint
 *   mjb_fwd_velocity           <- _src/forward.py:732  fwd_velocity (actuator velocity, com_vel, passive, rne)
 *   mjb_fwd_actuation          <- _src/forward.py:1152 fwd_actuation
 *   mjb_fwd_acceleration       <- _src/forward.py:1290 fwd_acceleration(factorize=True) (qfrc_smooth, factor M, qacc_smooth)
 *   mjb_factor_m               <- _src/smooth.py:1340  factor_m
 *   mjb_com_vel                <- _src/smooth.py:2261  com_vel
 *   mjb_passive                <- _src/passive.py:1257 passive (joint springs and dampers)
 *   mjb_rne                    <- _src/smooth.py:1499  rne(flg_acc=False)
 *   mjb_solve_m                <- _src/smooth.py:3214  solve_m(m, d, x, y): x = M^-1 y through Data.qLD
 *   mjb_mul_m                  <- _src/support.py:153  mul_m(m, d, res, vec): res = M vec
 *   mjb_sensor_pos/vel/acc     <- _src/sensor.py:810, :1432, :2512  sensor_pos / sensor_vel / sensor_acc(m, d)
 *   mjb_energy_pos/vel         <- _src/sensor.py:2934, :3004  energy_pos / energy_vel(m, d)
 *   mjb_read_ctrl / _sensor    <- _src/history.py:634, :718  read_ctrl / read_sensor(m, d, id, time, interp, result)
 *   mjb_init_ctrl_history /    <- _src/history.py:796, :881  init_ctrl_history(m, d, ctrlid, times, values) /
 *     mjb_init_sensor_history       init_sensor_history(m, d, sensorid, times, values, phase)
 *   mjb_contact_force          <- _src/support.py:445  contact_force(m, d, contact_ids, to_world_frame, force)
 *   mjb_rne_postconstraint     <- _src/smooth.py:1744  rne_postconstraint(m, d)
 *   mjb_subtree_vel            <- _src/smooth.py:3614  subtree_vel(m, d)
 *   mjb_tendon                 <- _src/smooth.py:4197  tendon(m, d) (fixed tendons: no wrap outputs)
 *   mjb_jac                    <- _src/support.py:583  jac(m, d, jacp, jacr, point, body)
 *   mjb_xfrc_accumulate        <- _src/support.py:314  xfrc_accumulate(m, d, qfrc)
 *   mjb_deriv_smooth_vel       <- _src/derivative.py:1117  deriv_smooth_vel(m, d, out)
 *   mjb_rays                   <- _src/ray.py:1219 rays(m, d, pnt, vec, geomgroup, flg_static, bodyexclude, dist, geomid, normal) without a
 *                                 render context (every geom tested, no BVH; no height fields)
 *   mjb_refit_bvh              <- _src/bvh.py:39 refit_bvh(m, d, rc): world-space bounds of the rendered geoms (no BVH is built;
 *                                 the renderer culls every geom against its bounds)
 *   mjb_render                 <- _src/render.py:656 render(m, d, rc) without textures, skybox, splats or flex
 *   mjb_render_rays            <- _src/render_util.py:255 _build_rays (the precomputed rays of create_render_context)
 *   mjb_rungekutta4            <- _src/forward.py:523  rungekutta4(m, d)
 *   mjb_solve                  <- _src/solver.py:3671  solve
 *   mjb_euler                  <- _src/forward.py:387  euler (always the semi-implicit Euler update, whatever the model's integrator)
 *   mjb_implicit               <- _src/forward.py:578  implicit (integrator IMPLICIT: qLU = M - dt (qDeriv_smooth + d RNE / d qvel) in the
 *                                                      D-structure, LU solve, Data.qLU written; IMPLICITFAST: symmetric M - dt qDeriv, Cholesky;
 *                                                      then advance.  Error for Euler / RK4 models: the scratch is sized per integrator)
 *   mjb_ctrl_noise             <- _src/cli.py:103      _ctrl_noise (harness kernel, untimed in testspeed)
 *   mjb_set_const              <- _src/set_const.py:613-950 set_const_fixed / set_const_0 / set_const_spring / set_const(m, d, restore)
 *   mjb_set_length_range       <- _src/set_const.py:952 set_length_range(m, d, index)
 *
 * Conventions: plain pointers and sizes only (no torch / warp types).  All array pointers are DEVICE
 * pointers owned by the caller for the lifetime of the handle (borrowed, never freed here).  Layout is
 * the reference's world-major SoA (types.py:2230-2374): a Data field of per-world shape S is a contiguous
 * (nworld, *S) fp32 / int32 array.  Every call enqueues work on `stream` (a cudaStream_t cast to void*)
 * and returns immediately; 0 = ok, non-zero = error (see mjb_last_error).  No device synchronisation and
 * no allocation happen after mjb_data_finalize, so a call sequence is CUDA-graph capturable.
 * Runtime failures never raise: they set bits in Data.overflow exactly like the reference (types.py:149-176).
 */
#ifndef MJB200_H
#define MJB200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mjbModel mjbModel;
typedef struct mjbData mjbData;

/* ---- Model: build by name, then finalize.  Names are the reference's Model field names. */
mjbModel* mjb_model_create(void);
void mjb_model_destroy(mjbModel* m);
int mjb_model_set_int(mjbModel* m, const char* name, int value);
int mjb_model_set_float(mjbModel* m, const char* name, float value);
/* dev_ptr: device array shared by all worlds (nbatch must be 1) */
int mjb_model_set_array(mjbModel* m, const char* name, const void* dev_ptr, int nbatch);
/* per-world (batched) float field, the reference's `*` leading dimension (types.py:822-833, io.py:259-282): nbatch entries of
 * batch_stride floats each, world w reads entry w % nbatch.  May be called again after finalize (e.g. when a field is re-randomised
 * into a new buffer); integer tables cannot be batched. */
int mjb_model_set_array_batched(mjbModel* m, const char* name, const void* dev_ptr, int nbatch, int batch_stride);
int mjb_model_finalize(mjbModel* m);

/* ---- Data */
mjbData* mjb_data_create(int nworld, int nconmax, int naconmax, int njmax, int njmax_pad, int nv_pad);
void mjb_data_destroy(mjbData* d);
int mjb_data_set_array(mjbData* d, const char* name, void* dev_ptr);
/* optional sizes set before finalize: "njmax_nnz" = capacity of the CSR view of efc.J (models the reference treats as sparse, io.py:153) */
int mjb_data_set_int(mjbData* d, const char* name, int value);
int mjb_data_finalize(mjbData* d, const mjbModel* m);

/* ---- pipeline */
int mjb_step(const mjbModel* m, mjbData* d, void* stream);
int mjb_forward(const mjbModel* m, mjbData* d, void* stream);
/* inverse.py:148 inverse: fwd_position and fwd_velocity (with actuation and the factor of M, as forward), then at the given d.qacc:
 * efc_force / efc_state / efc_Ma, qfrc_constraint, solver_niter = 0, qfrc_inverse = qfrc_bias + M qacc - qfrc_passive - qfrc_constraint,
 * and the sensors.  With ENBL_INVDISCRETE (Euler unless eulerdamp is disabled, implicitfast) d.qacc is a discrete-time acceleration:
 * everything above uses its continuous-time counterpart, and d.qacc is left as it was.  Error for RK4 / implicit with ENBL_INVDISCRETE. */
int mjb_inverse(const mjbModel* m, mjbData* d, void* stream);
int mjb_fwd_position(const mjbModel* m, mjbData* d, void* stream);
int mjb_kinematics(const mjbModel* m, mjbData* d, void* stream);
int mjb_com_pos(const mjbModel* m, mjbData* d, void* stream);
int mjb_camlight(const mjbModel* m, mjbData* d, void* stream);
int mjb_crb(const mjbModel* m, mjbData* d, void* stream);
int mjb_transmission(const mjbModel* m, mjbData* d, void* stream);
int mjb_collision(const mjbModel* m, mjbData* d, void* stream);
int mjb_make_constraint(const mjbModel* m, mjbData* d, void* stream);
int mjb_fwd_velocity(const mjbModel* m, mjbData* d, void* stream);
int mjb_fwd_actuation(const mjbModel* m, mjbData* d, void* stream);
int mjb_fwd_acceleration(const mjbModel* m, mjbData* d, void* stream);
int mjb_factor_m(const mjbModel* m, mjbData* d, void* stream);
int mjb_com_vel(const mjbModel* m, mjbData* d, void* stream);
int mjb_passive(const mjbModel* m, mjbData* d, void* stream);
int mjb_rne(const mjbModel* m, mjbData* d, void* stream);
/* x, y, res, vec: device arrays (nworld, nv) fp32 */
int mjb_solve_m(const mjbModel* m, mjbData* d, float* x, const float* y, void* stream);
int mjb_mul_m(const mjbModel* m, mjbData* d, float* res, const float* vec, void* stream);
/* sensor.py:810 / :1432 / :2512: the sensors of one stage (forward and step already evaluate all of them after the solver) */
int mjb_sensor_pos(const mjbModel* m, mjbData* d, void* stream);
int mjb_sensor_vel(const mjbModel* m, mjbData* d, void* stream);
int mjb_sensor_acc(const mjbModel* m, mjbData* d, void* stream);
/* Stages that read a finished forward pass, one kernel launch each over every world (see the exceptions below), whatever the model's sensors or DSBL_SENSOR say:
 * smooth.py:1744 rne_postconstraint (Data.cacc, cfrc_int, cfrc_ext; contact and equality wrenches summed in pool / row order),
 * smooth.py:3614 subtree_vel (Data.subtree_linvel, subtree_angmom), smooth.py:4197 tendon (Data.ten_length, ten_J of the fixed tendons; no
 * launch without tendons). */
int mjb_rne_postconstraint(const mjbModel* m, mjbData* d, void* stream);
int mjb_subtree_vel(const mjbModel* m, mjbData* d, void* stream);
int mjb_tendon(const mjbModel* m, mjbData* d, void* stream);
/* support.py:583 jac: jacp / jacr (nworld, 3, nv) fp32 device (either may be NULL) = the translational / rotational Jacobian of point
 * (nworld, 3) fp32 on body (nworld) int32; columns of dofs that do not move the body are 0; a body id outside [0, nbody) gives NaN rows.
 * jac and xfrc_accumulate launch nothing for a model without dofs */
int mjb_jac(const mjbModel* m, mjbData* d, float* jacp, float* jacr, const float* point, const int* body, void* stream);
/* support.py:314 xfrc_accumulate: qfrc (nworld, nv) fp32 device += J^T Data.xfrc_applied, bodies summed in index order */
int mjb_xfrc_accumulate(const mjbModel* m, mjbData* d, float* qfrc, void* stream);
/* derivative.py:1117 deriv_smooth_vel: out (nworld, nC) fp32 device = M - dt qDeriv in Data.M's layout (M_rowadr / M_colind); qDeriv: affine
 * actuators (unless DSBL_ACTUATION), dof and tendon damping (unless DSBL_DAMPER), fluid forces (an ellipsoid's derivative symmetrized for the
 * implicitfast integrator only, as the reference does) */
int mjb_deriv_smooth_vel(const mjbModel* m, mjbData* d, float* out, void* stream);
/* sensor.py:2934 energy_pos / :3004 energy_vel: Data.energy[:, 0] = potential energy (gravity unless DSBL_GRAVITY; joint and fixed-tendon
 * springs unless DSBL_SPRING) at the last position stage; Data.energy[:, 1] = 1/2 qvel . M qvel with the M of the last crb.  Whatever
 * ENBL_ENERGY says; one kernel launch each.  Data.energy is bound by name ("energy", (nworld, 2) fp32).  forward / step / step1 compute
 * both terms when ENBL_ENERGY is set; the e_potential / e_kinetic sensors are written by mjb_sensor_pos, forward, step and inverse. */
int mjb_energy_pos(const mjbModel* m, mjbData* d, void* stream);
int mjb_energy_vel(const mjbModel* m, mjbData* d, void* stream);
/* history.py: actuator and sensor delays.  Data.history is bound by name ("history", (nworld, nhistory) fp32); the Model's delay fields
 * ("actuator_history" (nu, 2) int, "actuator_historyadr", "actuator_delay", "sensor_history", "sensor_historyadr", "sensor_delay",
 * "sensor_interval" (nsensor, 2), "sensor_history_id": the sensors with nsample > 0) and the ints "nhistory", "nactuator_history",
 * "nsensor_history" by name as well.  forward / step read the delayed ctrl in the actuation stage, replace delayed / interval sensors after
 * each sensor stage and insert d.ctrl once per step before time advances.
 * read_ctrl / read_sensor: the value of actuator / sensor `id` at time[w] - delay into result (nworld) / (nworld, sensor_dim), with interp
 * -1 (the model's), 0 zoh, 1 linear or 2 cubic; the current ctrl / sensordata for an id without a buffer.  init_*_history: the buffer of
 * `id` (which must have nsample > 0) from times (nsample, strictly increasing; NULL: -MJ_MAXVAL stamps) and values (nworld, nsample *
 * dim), newest last; a sensor's user slot becomes phase[w] (the last time an interval sensor was due), an actuator's is kept.  All
 * arrays are fp32 device pointers; one kernel launch each. */
int mjb_read_ctrl(const mjbModel* m, mjbData* d, int ctrlid, const float* time, int interp, float* result, void* stream);
int mjb_read_sensor(const mjbModel* m, mjbData* d, int sensorid, const float* time, int interp, float* result, void* stream);
int mjb_init_ctrl_history(const mjbModel* m, mjbData* d, int ctrlid, const float* times, const float* values, void* stream);
int mjb_init_sensor_history(const mjbModel* m, mjbData* d, int sensorid, const float* times, const float* values, const float* phase, void* stream);
/* support.py:445 contact_force(m, d, contact_ids, to_world_frame, force): force is (n, 6) floats, device pointers */
int mjb_contact_force(const mjbModel* m, mjbData* d, const int* contact_ids, int n, int to_world_frame, float* force, void* stream);
/* ray.py:1219 rays: pnt, vec (pnt_nbatch, nray, 3) fp32 device, pnt_nbatch 1 or nworld; geomgroup: 6 host ints (all -1 = no group
 * filter; NULL = all -1); bodyexclude (nray) int32 device; dist (nworld, nray) fp32, geomid (nworld, nray) int32, normal (nworld, nray, 3)
 * fp32.  Reads the geom poses of the last kinematics.  A miss gives dist -1, geomid -1 and a zero normal; among equally distant hits the
 * lowest geom id wins.  One kernel launch (none for nray = 0). */
int mjb_rays(const mjbModel* m, mjbData* d, const float* pnt, const float* vec, int nray, int pnt_nbatch, const int* geomgroup,
             int flg_static, const int* bodyexclude, float* dist, int* geomid, float* normal, void* stream);
/* The render context of mjb_refit_bvh / mjb_render (render_util.py:272 create_render_context; types.py RenderContext): the cameras
 * that render, their pixel buffers and the enabled geoms, plus the Model's camera, light and material fields the renderer reads.  All
 * pointers are device pointers.  A per-world Model field has nb_<field> entries (world w reads entry w % nb); 1 = shared. */
typedef struct mjbRender {
  int ncam;                      /* cameras that render (the context's active cameras) */
  int ngeom;                     /* enabled geoms (geom group filter) */
  int npixel;                    /* pixels of all active cameras */
  int nrgb, ndepth, nseg;        /* row lengths of rgb / depth / seg (pixels of the cameras that render each output) */
  const int* cam_id;             /* (ncam) Model camera id of each active camera */
  const int* cam_res;            /* (ncam, 2) width, height */
  const int* pix_adr;            /* (ncam) first pixel of each camera in the ray table */
  const int* rgb_adr;            /* (ncam) first pixel in rgb, -1: not rendered; depth_adr / seg_adr likewise */
  const int* depth_adr;
  const int* seg_adr;
  const float* ray;              /* (npixel, 3) camera-frame ray directions (use_precomputed_rays), else NULL */
  const int* geom_id;            /* (ngeom) enabled geom ids, ascending */
  const float* mesh_half;        /* (nmesh, 3) half-extent of each mesh's vertex box (the bounds of its geoms) */
  float* lower;                  /* (nworld, ngeom, 3) world-space bounds written by mjb_refit_bvh */
  float* upper;
  unsigned* rgb;                 /* (nworld, nrgb) packed 0xAARRGGBB */
  float* depth;                  /* (nworld, ndepth) planar depth */
  int* seg;                      /* (nworld, nseg, 2) geom id, object type */
  const int* cam_projection;     /* (ncam_model) */
  const float* cam_fovy;         /* (nb, ncam_model) */
  const float* cam_sensorsize;   /* (ncam_model, 2) */
  const float* cam_intrinsic;    /* (nb, ncam_model, 4) */
  int nb_cam_fovy, nb_cam_intrinsic;
  int nlight;
  const int* light_type;         /* (nlight) */
  const int* light_castshadow;
  const int* light_active;
  const float* light_attenuation; /* (nb, nlight, 3) */
  const float* light_cutoff;     /* (nb, nlight) degrees */
  const float* light_exponent;
  const float* light_ambient;    /* (nb, nlight, 3) */
  const float* light_diffuse;
  const float* light_specular;
  int nb_light_attenuation, nb_light_cutoff, nb_light_exponent, nb_light_ambient, nb_light_diffuse, nb_light_specular;
  const float* mat_specular;     /* (nb, nmat) */
  const float* mat_shininess;
  const float* mat_emission;
  int nb_mat_specular, nb_mat_shininess, nb_mat_emission;
  int use_shadows, use_ambient_lighting, enable_per_light_ambient, enable_specular, enable_emission, enable_backface_culling;
  int headlight_active, light_attenuation_is_default, has_spot_lights;
  unsigned background_color;     /* packed like rgb */
  float znear;
  float headlight_ambient[3], headlight_diffuse[3], headlight_specular[3];
} mjbRender;
/* render_util.py:255 _build_rays (create_render_context with use_precomputed_rays): ray (npixel, 3) receives the camera-frame ray of
 * every pixel of rc's active cameras, from entry 0 of cam_fovy / cam_intrinsic.  Needs rc's camera tables only.  One kernel launch. */
int mjb_render_rays(const mjbRender* rc, float* ray, void* stream);
/* bvh.py:39 refit_bvh: lower / upper of every enabled geom of every world from d.geom_xpos / geom_xmat (bvh.py:178 _compute_bvh_bounds,
 * with its 1000-unit extent for infinite planes).  One kernel launch. */
int mjb_refit_bvh(const mjbModel* m, mjbData* d, const mjbRender* rc, void* stream);
/* render.py:656 render: one image per (world, active camera) into rc's rgb / depth / seg.  Reads geom_xpos / geom_xmat, cam_xpos /
 * cam_xmat and light_xpos / light_xdir of the last kinematics and the bounds of the last mjb_refit_bvh; writes no Data field.  Each pixel
 * casts its primary ray against every enabled geom whose bounds it enters (closest hit; equal distances go to the lower geom id), shades
 * it with emission, ambient, every light's diffuse / specular term and the headlight, and with use_shadows casts a shadow ray per light.
 * A miss writes background_color, depth 0 and (-1, -1).  One kernel launch. */
int mjb_render(const mjbModel* m, mjbData* d, const mjbRender* rc, void* stream);
/* forward.py:523 rungekutta4(m, d): the integrator alone, after forward() (models compiled with the RK4 integrator) */
int mjb_rungekutta4(const mjbModel* m, mjbData* d, void* stream);
int mjb_solve(const mjbModel* m, mjbData* d, void* stream);
int mjb_euler(const mjbModel* m, mjbData* d, void* stream);
int mjb_implicit(const mjbModel* m, mjbData* d, void* stream);
/* set_const.py:613-950: recompute the Model fields the compiler derives from other Model fields.  parts is a combination of
 *   MJB_SET_CONST_FIXED   body_subtreemass from body_mass (set_const_fixed);
 *   MJB_SET_CONST_0       at qpos0: stat.meaninertia, tendon_length0, eq_data (connect / weld), dof_invweight0, body_invweight0,
 *                         tendon_invweight0, cam_pos0 / poscom0 / mat0, light_pos0 / poscom0 / dir0, actuator_acc0 and the dampratio
 *                         form of affine-bias actuators in actuator_biasprm[2] (set_const_0);
 *   MJB_SET_CONST_SPRING  at qpos_spring: tendon_lengthspring entries that are (-1, -1) (set_const_spring; nothing without tendons);
 * all three is set_const.  Entry i of a derived field with a leading (batch) size nb is computed from world i, for i < nb (unbatched: world
 * 0); an output with nb > nworld is an error.  stat.meaninertia stays a Model scalar: world 0's value is written to the device array bound
 * as "meaninertia" (mjb_model_set_array), and the caller hands it to mjb_model_set_float once it has read it back.  "actuator_acc0" is
 * bound by name like the other arrays (batched like a float field).  d.qpos is restored bit-exactly; with restore, the position stages
 * and the factor of M are recomputed at it for every world, otherwise the worlds that were evaluated keep the state at qpos0 / qpos_spring.
 * Stream-ordered, no allocation, no synchronisation; the number of kernels depends on parts and restore only. */
#define MJB_SET_CONST_FIXED 1
#define MJB_SET_CONST_0 2
#define MJB_SET_CONST_SPRING 4
int mjb_set_const(const mjbModel* m, mjbData* d, int parts, int restore, void* stream);
/* set_const.py:573-607, 952-985: actuator_lengthrange from the joint and tendon limits.  An actuator on a limited joint or limited fixed
 * tendon gets the limit range times gear[0] (ends swapped for a negative gear); every other actuator gets (0, 0).  Every actuator is
 * written whatever index is, as the reference does; index must be -1 or an actuator id.  Entry i of a batched actuator_lengthrange is
 * computed from world i (jnt_range / tendon_range / gear read as world i sees them); nb > nworld is an error.  One kernel, stream-ordered. */
int mjb_set_length_range(const mjbModel* m, mjbData* d, int index, void* stream);
/* ctrl <- OU noise around ctrl_center (device array of nu floats, or NULL), reference cli.py:103-145 */
int mjb_ctrl_noise(const mjbModel* m, mjbData* d, const float* ctrl_center, int step, float noise_std, float noise_rate, void* stream);

/* profiling aid: runs ONE step's kernel chain over all worlds on `stream` (not split over world halves), synchronises, and writes
 * the durations in ms of its 6 stage groups to ms_out (host pointer, 6 floats): position, collision, constraint (with the CSR
 * view of sparse models), velocity, solver (with the sensors), integrate (every integrator kernel).  The contact-counter resets
 * run before the first event, so the durations cover kernels only.  RK4 models profile one forward pass and the Euler update. */
int mjb_step_profile(const mjbModel* m, mjbData* d, void* stream, float* ms_out);

/* worlds per SM that are resident at once (cudaOccupancyMaxActiveBlocksPerMultiprocessor times worlds per block) in the launch
 * shape k_position / k_velocity take for all of d's worlds.  Both kernels are latency bound: they finish in
 * ceil(nworld / (SMs x worlds per SM)) rounds of one world's dependent chain.  shapes (host pointer to 8 ints, or NULL) receives the
 * launch shape behind each count, k_position's in shapes[0..3] and k_velocity's in shapes[4..7]: lanes per world (8, 16 or 32), warps
 * per block, shared-memory bytes per block, and the instance (k_velocity: 0 plain, 1 with gravity compensation / ball and free joint
 * springs / tendons, 2 with fluid forces; k_position: 0). */
int mjb_team_residency(const mjbModel* m, const mjbData* d, int* position_worlds, int* velocity_worlds, int* shapes);

/* name of the collision kernel m's collision stage launches: "k_collision" (no mesh geoms), "k_collision_mesh", or "k_collision_mesh_large"
 * (a hull polygon of more than 32 vertices or a hull vertex in more than 16 polygons: model-sized multi-contact buffers in global scratch,
 * and the collision sensors' kernel built the same way); null with mjb_last_error set if m is not finalized */
const char* mjb_collision_kernel(const mjbModel* m);

/* number of kernels launched by the calling thread's last mjb_* call that enqueues work, counted at each launch (memsets are not
 * kernels and are not counted); bench.py's gpu_launches */
int mjb_last_launch_count(void);
const char* mjb_last_error(void);
const char* mjb_version(void);

#ifdef __cplusplus
}
#endif
#endif
