/* mjb200.h -- C ABI of the H100-native (sm_90a) batched MuJoCo physics step (libmjb200.so).
 *
 * Drop-in boundary for the step path of google-deepmind/mujoco_warp.  Every entry point replaces a
 * Python function of the reference's public API (paths relative to /root/reference/mujoco_warp/):
 *
 *   mjb_model_* / mjb_data_*   <- _src/io.py:259 put_model, :1680 make_data, :1890 put_data (device SoA binding;
 *                                 the reference binds wp.array pointers into wp.launch argument lists)
 *   mjb_step                   <- _src/forward.py:1368 step(m, d)
 *   mjb_forward                <- _src/forward.py:1341 forward(m, d)
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
 *   mjb_contact_force          <- _src/support.py:445  contact_force(m, d, contact_ids, to_world_frame, force)
 *   mjb_rungekutta4            <- _src/forward.py:523  rungekutta4(m, d)
 *   mjb_solve                  <- _src/solver.py:3671  solve
 *   mjb_euler                  <- _src/forward.py:387  euler (always the semi-implicit Euler update, whatever the model's integrator)
 *   mjb_implicit               <- _src/forward.py:578  implicit (integrator IMPLICIT: qLU = M - dt (qDeriv_smooth + d RNE / d qvel) in the
 *                                                      D-structure, LU solve, Data.qLU written; IMPLICITFAST: symmetric M - dt qDeriv, Cholesky;
 *                                                      then advance.  Error for Euler / RK4 models: the scratch is sized per integrator)
 *   mjb_ctrl_noise             <- _src/cli.py:103      _ctrl_noise (harness kernel, untimed in testspeed)
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
/* support.py:445 contact_force(m, d, contact_ids, to_world_frame, force): force is (n, 6) floats, device pointers */
int mjb_contact_force(const mjbModel* m, mjbData* d, const int* contact_ids, int n, int to_world_frame, float* force, void* stream);
/* forward.py:523 rungekutta4(m, d): the integrator alone, after forward() (models compiled with the RK4 integrator) */
int mjb_rungekutta4(const mjbModel* m, mjbData* d, void* stream);
int mjb_solve(const mjbModel* m, mjbData* d, void* stream);
int mjb_euler(const mjbModel* m, mjbData* d, void* stream);
int mjb_implicit(const mjbModel* m, mjbData* d, void* stream);
/* ctrl <- OU noise around ctrl_center (device array of nu floats, or NULL), reference cli.py:103-145 */
int mjb_ctrl_noise(const mjbModel* m, mjbData* d, const float* ctrl_center, int step, float noise_std, float noise_rate, void* stream);

/* profiling aid: runs ONE step with a CUDA-event pair around each of the 6 kernels (position, collision, constraint,
 * velocity, solver, integrate), synchronises, and writes the 6 durations in ms to ms_out (host pointer). */
int mjb_step_profile(const mjbModel* m, mjbData* d, void* stream, float* ms_out);

/* number of kernels the last mjb_* pipeline call launched (for bench.py's gpu_launches) */
int mjb_last_launch_count(void);
const char* mjb_last_error(void);
const char* mjb_version(void);

#ifdef __cplusplus
}
#endif
#endif
