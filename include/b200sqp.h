/*
 * b200sqp -- C ABI of the GPU-native (H100, sm_90a) batched multiple-shooting SQP solver.
 *
 * This is the drop-in boundary for ONE hot path of manumerous/wb_humanoid_mpc: the SQP iteration
 * ocs2::SqpSolver::runImpl (lib/ocs2_ros2/ocs2_sqp/ocs2_sqp/src/SqpSolver.cpp:193-284) for the Unitree G1
 * whole-body optimal-control problem, batched over independent MPC instances.  Plain pointers and sizes only;
 * no C++/torch types cross this boundary.  Every entry point names the reference interface it replaces.
 *
 * Conventions
 *   - return 0 on success, a negative B200SQP_E* code on failure; nothing throws across the ABI;
 *     b200sqp_last_error() returns a human-readable reason for the last failure on this thread.
 *   - all matrices are column-major fp64 (Eigen's default, as in ocs2 VectorFunctionLinearApproximation /
 *     ScalarFunctionQuadraticApproximation, ocs2_core/include/ocs2_core/Types.h:145-157,234-240).
 *   - the caller owns every host buffer; a handle owns its device memory; one handle per GPU;
 *     handles are thread-compatible (external synchronisation), like ocs2::SqpSolver (MPC_BASE.h:58).
 *   - there is no CPU fallback: every entry point that computes fails with B200SQP_ENODEV without a CUDA device.
 */
#ifndef B200SQP_H
#define B200SQP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SQP_OK 0
#define B200SQP_EINVAL -1   /* bad argument / size mismatch (ocs2 throws std::runtime_error on size checks) */
#define B200SQP_ENODEV -2   /* no CUDA device / CUDA runtime error */
#define B200SQP_ENOMEM -3
#define B200SQP_EQP -4      /* QP failed for at least one instance: "[SqpSolver] Failed to solve QP" (SqpSolver.cpp:306-308) */
#define B200SQP_ESTATE -5   /* call order violated (e.g. solve before upload) */

const char* b200sqp_last_error(void);
/* library / build information, e.g. "b200sqp 0.1 (sm_90a, fp64)" */
const char* b200sqp_version(void);

/* ------------------------------------------------------------------------------------------------------------------
 * (1) Batched QP sub-problem: replaces ocs2::HpipmInterface
 *     (lib/ocs2_ros2/ocs2_sqp/hpipm_catkin/include/hpipm_catkin/HpipmInterface.h; src/HpipmInterface.cpp:92-455).
 *
 *     minimise  sum_k 1/2 [dx;du]'[Q S';S R][dx;du] + q'dx + r'du   s.t.  dx_{k+1} = A dx + B du + b,  dx_0 given
 *
 *     Stage arrays are padded to nu_max inputs; stage k of instance i uses the leading nu[i*N+k] columns/rows
 *     (nu = 0 is the event-node shape of HpipmInterface test "noInputs", testHpipmInterface.cpp:208-256).
 *       A [B][N][nx*nx]        B [B][N][nx*nu_max]      b [B][N][nx]
 *       Q [B][N+1][nx*nx]      S [B][N][nu_max*nx] (leading dimension nu_max, = dfdux)
 *       R [B][N][nu_max*nu_max]  q [B][N+1][nx]         r [B][N][nu_max]
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_qp_t* b200sqp_qp;

/* HpipmInterface::HpipmInterface(OcpSize) / resize(): allocate device storage for `batch` problems of N stages.
 * Accepts 0 < nx <= 64 and 0 < nu_max <= 32 whose Riccati working set fits one block's shared memory in both kernel variants (1948 of the
 * 2048 pairs; the largest nu_max for nx = 64 is 15); B200SQP_EINVAL otherwise. */
int b200sqp_qp_create(int device, int batch, int N, int nx, int nu_max, b200sqp_qp* out);
void b200sqp_qp_destroy(b200sqp_qp qp);

/* HpipmInterface::solve(x0, dynamics, cost, nullptr, ...): host -> device copy of the LQ data. nu may be NULL (all nu_max). */
int b200sqp_qp_upload(b200sqp_qp qp, const double* A, const double* B, const double* b, const double* Q, const double* S,
                      const double* R, const double* q, const double* r, const int32_t* nu, const double* dx0);

/* d_ocp_qp_ipm_solve for the unconstrained QP: one backward Riccati factorisation + forward substitution, all instances.
 * reg_prim is added to the Hessian diagonals (hpipm_catkin HpipmInterfaceSettings.h:45-56, default 1e-12).
 * Asynchronous on `stream` (a cudaStream_t, may be NULL). keep_P != 0 stores the cost-to-go for b200sqp_qp_download. */
int b200sqp_qp_solve(b200sqp_qp qp, double reg_prim, int keep_P, void* stream);

/* getStateSolution/getInputSolution, getRiccatiFeedback, getRiccatiFeedforward, getRiccatiCostToGo.
 *   dx [B][N+1][nx], du [B][N][nu_max], K [B][N][nu_max*nx] (ld nu_max), k [B][N][nu_max], P [B][N+1][nx*nx], p [B][N+1][nx],
 *   status [B] (0 ok, 1 = Cholesky failed / NaN -> hpipm_status != SUCCESS).  Any pointer may be NULL.  Synchronises. */
int b200sqp_qp_download(b200sqp_qp qp, double* dx, double* du, double* K, double* k, double* P, double* p, int32_t* status);

/* device-time of the last b200sqp_qp_solve in milliseconds (CUDA events on the launching stream) */
int b200sqp_qp_last_ms(b200sqp_qp qp, float* ms);

/* ------------------------------------------------------------------------------------------------------------------
 * (2) Whole-body SQP solver: replaces ocs2::SqpSolver for the humanoid whole-body OCP
 *     (SqpSolver.h:60-103; OCP wiring humanoid_nmpc/humanoid_wb_mpc/src/WBMpcInterface.cpp:131-199).
 * ------------------------------------------------------------------------------------------------------------------ */
#define B200SQP_MAX_BODIES 32
#define B200SQP_MAX_FRAMES 16

/* Model constants the reference keeps inside PinocchioInterface + ModelSettings + the cost/constraint objects;
 * produced from URDF + task.info by wb_humanoid_mpc_b200/model_loader.py (or any caller that fills the arrays). */
typedef struct b200sqp_model_desc {
  int32_t nj;                                  /* actuated joints (23 for G1); nx = 2*(6+nj), nu = 12+nj */
  int32_t parent[B200SQP_MAX_BODIES];          /* parent body of body i (body 0 = floating base, parent -1) */
  double joint_R[B200SQP_MAX_BODIES][9];       /* row-major rotation of the joint frame in the parent body frame */
  double joint_p[B200SQP_MAX_BODIES][3];
  double joint_axis[B200SQP_MAX_BODIES][3];    /* revolute axis in the joint frame */
  double mass[B200SQP_MAX_BODIES];
  double com[B200SQP_MAX_BODIES][3];
  double inertia[B200SQP_MAX_BODIES][9];       /* rotational inertia about the com, body axes, row-major */
  double q_lower[B200SQP_MAX_BODIES], q_upper[B200SQP_MAX_BODIES]; /* index = joint (0-based) */
  int32_t n_frames;                            /* operational frames: [0..2] left foot contact, p1, p2; [3..5] right; 6,7 ankles; 8,9 knees */
  int32_t frame_body[B200SQP_MAX_FRAMES];
  double frame_p[B200SQP_MAX_FRAMES][3];
  double gravity;
  double contact_rect[4];                      /* x_min, x_max, y_min, y_max (task.info contacts.contact_rectangle) */
  double Q_diag[64], R_diag[48], Qf_diag[64];  /* StateInputQuadraticCost / terminal cost weights (task.info Q, R, Q_final*scaling) */
  double foot_gain_pos_z, foot_gain_ori, foot_gain_linvel_z, foot_gain_linvel_xy, foot_gain_angvel, foot_gain_linacc_z,
      foot_gain_linacc_xy, foot_gain_angacc;   /* model_settings.foot_constraint */
  double foot_cost_w[18];                      /* EndEffectorDynamicsWeights::toVector() as actually loaded */
  double fric_coeff, fric_mu, fric_delta, fric_reg, fric_hess_shift; /* FrictionForceConeConstraint + RelaxedBarrierPenalty */
  double momxy_mu, momxy_delta;                /* ContactMomentXY relaxed barrier */
  double jlim_mu, jlim_delta;                  /* JointLimitsSoftConstraint piecewise-polynomial barrier */
  double coll_mu, coll_delta, coll_r_foot, coll_r_knee; /* FootCollisionConstraint */
  int32_t arm_swing_joint[4];                  /* l shoulder, r shoulder, l elbow, r elbow joint indices */
} b200sqp_model_desc;

/* sqp::Settings fields the hot path reads (ocs2_sqp/include/ocs2_sqp/SqpSettings.h:40-87) */
typedef struct b200sqp_settings {
  int32_t sqp_iteration;       /* sqpIteration */
  double delta_tol, cost_tol;  /* deltaTol, costTol */
  double alpha_decay, alpha_min, gamma_c, g_max, g_min, armijo_factor;
  double reg_prim;             /* HPIPM reg_prim */
  int32_t use_feedback_policy; /* useFeedbackPolicy: compute remapped K (toPrimalSolution, SqpSolver.cpp:331-344) */
  int32_t global_step;         /* 0: per-instance line search (reference semantics); 1: one step size for the whole (multi-GPU) batch */
  int32_t create_value_function; /* createValueFunction: keep the Riccati cost-to-go (extractValueFunction, SqpSolver.cpp:321-329) */
} b200sqp_settings;
void b200sqp_default_settings(b200sqp_settings* s);

typedef struct b200sqp_solver_t* b200sqp_handle;

/* Longest back-tracking ladder a handle serves: alpha_decay 0.95 with alpha_min 1e-4 takes 180 trials. */
#define B200SQP_MAX_LS_TRIALS 200

/* Number of trials of SqpSolver::takeStep's back-tracking (SqpSolver.cpp:527-565) for these settings: alpha = 1 is always tried (a do-while
 * loop), then alpha *= alpha_decay -- by repeated multiplication -- while alpha >= alpha_min.  B200SQP_EINVAL, with a message, for settings
 * b200sqp_create and b200sqp_cen_create reject: sqp_iteration outside [1, 1000]; a non-finite delta_tol, cost_tol, alpha_decay, alpha_min,
 * gamma_c, g_max, g_min or armijo_factor; alpha_decay outside (0, 1); alpha_min <= 0; more than B200SQP_MAX_LS_TRIALS trials; more than 32
 * trials with global_step = 1 (the candidates of the global-step mode, b200sqp_global_stats).  Needs no device. */
int b200sqp_line_search_trials(const b200sqp_settings* settings, int32_t* n_trials);

/* SqpSolver::SqpSolver(settings, ocp, initializer); the settings as b200sqp_line_search_trials checks them */
int b200sqp_create(const b200sqp_model_desc* model, const b200sqp_settings* settings, int device, b200sqp_handle* out);
void b200sqp_destroy(b200sqp_handle h);

/* batch of `batch` instances with n_nodes shooting nodes each (N = n_nodes-1 intervals incl. event nodes) */
int b200sqp_set_batch(b200sqp_handle h, int batch, int n_nodes);

/* Per-instance inputs of one runImpl call, i.e. what SolverBase::preRun + initializeStateInputTrajectories produce on the host:
 *   x0 [B][nx]; x_init [B][n_nodes][nx], u_init [B][n_nodes-1][nu] (warm start / WeightCompInitializer);
 *   t_nodes [B][n_nodes]; node_event [B][n_nodes] (0 none, 1 PreEvent, 2 PostEvent: AnnotatedTime::Event);
 *   contact_flags [B][n_nodes][2]; swing_ref [B][n_nodes][2][3] (swing-z position, velocity, acceleration);
 *   impact_factor [B][n_nodes][2]; arm_phase [B][n_nodes] (sin(2 pi (phase-0.15)), SwitchedModelReferenceManager.cpp:110-135);
 *   x_ref [B][n_nodes][nx] (TargetTrajectories::getDesiredState at node times). */
int b200sqp_upload_instances(b200sqp_handle h, const double* x0, const double* x_init, const double* u_init, const double* t_nodes,
                             const uint8_t* node_event, const uint8_t* contact_flags, const double* swing_ref,
                             const double* impact_factor, const double* arm_phase, const double* x_ref);

/* Page-locked host staging memory for the upload / download arrays (plain malloc-like interface so that hosts without CUDA headers can use
 * it); NULL on failure.  Arrays passed to b200sqp_upload_instances / b200sqp_download may live anywhere; pinned ones copy faster. */
void* b200sqp_host_alloc(size_t bytes);
void b200sqp_host_free(void* p);

/* SqpSolver::reset() (SqpSolver.h:62): drop the current iterate; the next solve starts again from the uploaded initial guess
 * (device-to-device restore, no host traffic). */
int b200sqp_reset(b200sqp_handle h);

/* SqpSolver::runImpl for every instance, ASYNCHRONOUS on `stream` (NULL = the legacy default stream): every kernel of up to sqp_iteration SQP
 * iterations is enqueued and the call returns; nothing on the host waits for the device.  The filter line search needs no host decision: an
 * instance needs at most b200sqp_line_search_trials trials (14 with the default settings), all of them are enqueued, and the thread blocks of
 * an instance whose search has ended return at their first instruction (likewise every kernel for a converged instance).  b200sqp_wait -- or
 * any entry point that reads results or re-uses the handle (download*, get_stage_times, reset, upload / build_instances, set_batch, destroy) --
 * waits for the stream first.  One solve per handle in flight; several handles on several streams overlap on the device.  (The global-step mode takes a
 * host decision per candidate step and returns when the solve has finished.) */
int b200sqp_solve(b200sqp_handle h, void* stream);
/* Blocks until the last b200sqp_solve of this handle has finished; reports CUDA errors of the asynchronous work. */
int b200sqp_wait(b200sqp_handle h);

/* A non-blocking CUDA stream owned by the handle, for callers without CUDA headers: b200sqp_solve(h, stream) on it lets several handles
 * (e.g. two b200sqp::host::SqpSolver objects double-buffering a workload) overlap on the device instead of serialising on the legacy
 * default stream.  The handle's host<->device copies (upload / reset / download) run on a second internal stream and are complete when
 * those calls return. */
int b200sqp_own_stream(b200sqp_handle h, void** stream);

/* Global-step mode (settings.global_step = 1; SURVEY.md section 8e, not a reference semantic -- the reference searches per instance,
 * SqpSolver.cpp:517-565): one line-search step size per SQP iteration for the whole, possibly multi-GPU, batch.  Per iteration b200sqp_solve
 * walks the fixed ladder of the back-tracking trials (b200sqp_line_search_trials; at most 32 in this mode) from the largest candidate: one
 * roll-out of every active instance, the reference's filter test (FilterLinesearch.cpp:34-57), and
 *   stats[j] = { #instances that accept alpha_j, sum of their trial merits, max trial constraint violation, #active instances }
 * combined over all ranks by two NCCL all-reduces (4 doubles SUM + 1 double MAX, on `stream`) when a communicator has been set; it stops at
 * the first candidate every active instance of every rank accepts and applies it (a zero step when none is).  Every rank takes the same
 * decisions from the same reduced numbers.
 *
 * b200sqp_set_comm: the ncclComm_t of this process' rank (created by the caller with ncclCommInitRank; void* so that hosts without nccl.h
 * can forward it), n_ranks = its size.  NULL / 1 = single process.  The library resolves libnccl.so.2 at run time.
 * b200sqp_global_stats: combined statistics of the last iteration of the last solve, stats [32][4]; candidates [0, n_evaluated) were
 * evaluated; chosen = index of the applied candidate or -1. */
int b200sqp_set_comm(b200sqp_handle h, void* nccl_comm, int n_ranks);
int b200sqp_global_stats(b200sqp_handle h, double* stats /* [32][4] */, int32_t* n_evaluated, int32_t* chosen);
int b200sqp_global_ladder(b200sqp_handle h, double* alpha /* [32] */, int32_t* n_alpha);

/* ------------------------------------------------------------------------------------------------------------------
 * Device-side instance builder (SURVEY.md section 8(f)-1): what SolverBase::preRun + the top of SqpSolver::runImpl compute per instance on the
 * host -- SwitchedModelReferenceManager::modifyReferences (GaitSchedule::getModeSchedule, SwingTrajectoryPlanner::update), the velocity-command
 * target trajectories (WBMpcTargetTrajectoriesCalculator.cpp:82-136), timeDiscretizationWithEvents, initializeStateInputTrajectories with the
 * WeightCompInitializer -- evaluated on the GPU from a few numbers per instance.  b200sqp_build_instances replaces
 * b200sqp_upload_instances for batches whose instances share the horizon [t0, t0 + horizon] (a batch of synchronous MPC cycles).
 * Whole-body and centroidal handles (b200sqp_cen_create) are both served; on a centroidal handle the target trajectories follow
 * CentroidalMpcTargetTrajectoriesCalculator.cpp:86-160 (normalized momentum, base pose, default joints), whose base velocity Ab^-1 hbar of the
 * measured state is evaluated on the device with the handle's own centroidal model.
 * ------------------------------------------------------------------------------------------------------------------ */
#define B200SQP_MAX_GAITS 16
#define B200SQP_MAX_GAIT_MODES 8
typedef struct b200sqp_builder_desc {
  int32_t n_gaits;
  int32_t gait_n_modes[B200SQP_MAX_GAITS];                            /* ModeSequenceTemplate::modeSequence length (gait.info) */
  int32_t gait_modes[B200SQP_MAX_GAITS][B200SQP_MAX_GAIT_MODES];      /* 0 FLY, 1 RF, 2 LF, 3 STANCE (MotionPhaseDefinition.h) */
  double gait_switching_times[B200SQP_MAX_GAITS][B200SQP_MAX_GAIT_MODES + 1];
  double swing[8];                /* swing_trajectory_config: liftOffVelocity, touchDownVelocity, swingHeight, touchDownHeightOffset, swingTimeScale,
                                     impactProximityFactor lift-off velocity, touch-down velocity, mid-point value (task.info:64-74) */
  double default_joint_state[B200SQP_MAX_BODIES];                     /* reference.info defaultJointState */
  double total_mass;
  double dt;                      /* sqp dt */
} b200sqp_builder_desc;
int b200sqp_set_builder(b200sqp_handle h, const b200sqp_builder_desc* desc);

/* One synchronous MPC cycle of `batch` instances (whole-body or centroidal) over [t0, t0 + horizon]:
 *   x0 [B][nx] measured states (nx = 58 whole-body, 12 + nj = 35 centroidal, as every state array of the handle's ABI);
 *   gait [B] index into the gait table (its template is tiled from gait_start[b] <= 0.5, STANCE before; the table's "stance" template
 *   reproduces the default schedule of GaitSchedule); cmd [B][4] = (v_x, v_y, pelvis height, yaw rate).
 *   warm = 0: cold start (x_k = x0, WeightCompInitializer inputs); warm = 1: the iterate left on the device by the previous solve of this
 *   handle is the previous primal solution and is shifted by the reference's rule (Initialization.cpp:35-79) -- no host copy of x / u.
 *   With warm = 1, x0 may be NULL: the measured state is then the previous plan interpolated at t0 on the device (perfect tracking, the dummy
 *   simulation of the reference's launch files), which closes the MPC loop without any per-cycle state transfer.
 *   warm = 2: warm start as with warm = 1, the measured state being the simulated state of the last b200sqp_rollout_policy of this batch (x0 must
 *   be NULL; B200SQP_ESTATE without such a roll-out): the closed loop of the reference's dummy simulation (MPC, roll-out, MPC, ...) on the device.
 *   On a centroidal handle the roll-out is b200sqp_cen_rollout_policy; the padding of the simulated state stays zero.
 * Every instance must produce the same number of shooting nodes (same event count inside the horizon); *n_nodes returns it, B200SQP_EINVAL
 * otherwise (group such instances by gait phase on the host).  Host pointers; ~0.5 kB per instance cross PCIe. */
int b200sqp_build_instances(b200sqp_handle h, int batch, double t0, double horizon, const double* x0, const int32_t* gait, const double* gait_start,
                            const double* cmd, int warm, int32_t* n_nodes);

/* The per-instance inputs as they currently lie on the device (the arrays of b200sqp_upload_instances, whoever produced them: the upload or the
 * device-side builder), e.g. to log the references a batch was solved with.  x_init / u_init are the initial guess (what b200sqp_reset restores).
 * Layout of b200sqp_upload_instances (on a centroidal handle x0, x_init and x_ref have nx = 12 + nj).  Any pointer may be NULL. */
int b200sqp_download_instances(b200sqp_handle h, double* x0, double* x_init, double* u_init, double* t_nodes, uint8_t* node_event, uint8_t* contact_flags,
                               double* swing_ref, double* impact_factor, double* arm_phase, double* x_ref);

/* Gait changes in the device-resident loop.  stateful = 0 (the default): every build recomputes each instance's schedule in closed form from
 * (gait, gait_start) and the warm start interpolates the previous solution as it is.  stateful = 1: each instance keeps its GaitSchedule on the
 * device across cycles (GaitSchedule::getModeSchedule every build), and the gait[] of a warm b200sqp_build_instances is the per-instance gait
 * command: a value different from the instance's last command runs GaitScheduleUpdater::updateGaitSchedule after this cycle's schedule was
 * taken (the reference manager runs before the synchronized modules), so it shows in the next cycle's schedule.  The warm start then applies
 * trajectorySpread(old schedule, new schedule, previous solution) first, as SqpSolver::runImpl does.  gait_start[] is used by cold builds only;
 * phase_transition_stance_time is GaitSchedule's phaseTransitionStanceTime (0.0 in the G1 task.info).  A change of mode or of
 * phase_transition_stance_time takes effect at the next cold build; a warm build after a change of mode returns B200SQP_ESTATE, and so does
 * a warm build after a failed stateful warm build (its schedules were already advanced).  B200SQP_ESTATE while a fleet is attached (set it
 * before b200sqp_fleet_create).  Centroidal handles (they have b200sqp_cen_set_gait_schedule), negative or non-finite times: B200SQP_EINVAL. */
int b200sqp_set_gait_schedule(b200sqp_handle h, int stateful, double phase_transition_stance_time);
/* b200sqp_set_gait_schedule for a centroidal handle (b200sqp_cen_create), with the same arguments, rules and error codes: the stateful schedule,
 * GaitScheduleUpdater and trajectorySpread are the same functions on both families.  Whole-body handles: B200SQP_EINVAL. */
int b200sqp_cen_set_gait_schedule(b200sqp_handle h, int stateful, double phase_transition_stance_time);

/* Joint-torque cost of the whole-body OCP: the reference's JointTorqueCostCppAd (getJointTorqueCost(taskFile) added to the cost collection).
 * weights [nj], MPC joint order (task.info joint_torque_weights): every intermediate node -- not PreEvent nodes, not the terminal node -- gets the
 * Gauss-Newton cost 1/2 |sqrt(w) .* tau(x, u)|^2 with tau = computeJointTorques(x, u) (the map of b200sqp_joint_torques, evaluated with the
 * instance's own MPC model: the handle's, or its B200SQP_PARAMS_MODEL record), scaled by the node's dt in the LQ approximation and in every
 * line-search trial, like the other costs.  NULL or all-zero weights turn the term off (the default): the solve is then the same kernels and
 * launches as without this call.  Takes effect at the next solve, for every instance, on the upload and the builder path alike; synchronous.
 * Centroidal handles, a negative or non-finite weight: B200SQP_EINVAL, and nothing is applied.  B200SQP_ESTATE while a fleet is attached
 * (set it before b200sqp_fleet_create). */
int b200sqp_set_joint_torque_cost(b200sqp_handle h, const double* weights /* [nj] or NULL */);

/* The window mode schedule [t0 - T, tf + T] the last b200sqp_build_instances used, in either mode: event_times [B][max_events],
 * mode_sequence [B][max_events + 1] (modes after the n_events[b] + 1 used entries are -1), n_events [B].  B200SQP_EINVAL when an instance has
 * more than max_events events. */
int b200sqp_download_mode_schedule(b200sqp_handle h, int max_events, double* event_times, int32_t* mode_sequence, int32_t* n_events);

/* Automatic gait selection: ProceduralMpcMotionManager::preSolverRun (humanoid_common_mpc/src/reference_manager/ProceduralMpcMotionManager.cpp:
 * 119-160), the only synchronized module of the reference's SQP nodes, per instance on the device.  Whole-body handles in the stateful mode
 * (centroidal handles: b200sqp_cen_set_motion_manager below).
 * With a manager, cmd [B][4] of every build is the raw WalkingVelocityCommand message (v_x, v_y, pelvis height, yaw rate): it is clamped to
 * [-1, 1] / [0.2, 1] (getWalkingVelocityCommandFromMsg), scaled by the three reference.info maxima below (the height is not scaled) and
 * filtered by the reference's BreakFrequencyAlphaFilter(5 Hz, 0), which never updates its last output or call time: the filtered command is
 * alpha * scaled with alpha = dt / (dt + 1 / (2 pi 5)), dt the time since construction.  dt is measured in MPC time, t0 - filter_origin
 * (the reference reads steady_clock).  The filtered command gives the target trajectories (commandedVelocityToTargetTrajectories, with the
 * build's t0, tf and x0), which go to the reference manager's buffer: the targets of a warm build are those computed by the previous build
 * (ReferenceManager::preSolverRun copies the buffer in before the synchronized modules run); a cold build uses its own.  After the 0.2 s hold
 * (t0 > last change + 0.2, the last change starting at 0.0) one band transition of the state machine stance, slow_walk, walk, slower_trot,
 * slow_trot, trot, run (the band table of ProceduralMpcMotionManager.h:110-118) may fire on the filtered command and the measured base
 * velocity x0[nv .. nv + 6); a changed gait goes through updateGaitSchedule as a changed gait command of b200sqp_set_gait_schedule does.
 *   b200sqp_set_motion_manager: gait[7] = the builder gait ids of the seven states; md = NULL switches the manager off.  Like
 *   b200sqp_set_gait_schedule it takes effect at the next cold build and a warm build after a change returns B200SQP_ESTATE.  B200SQP_ESTATE
 *   while a fleet is attached (set it before b200sqp_fleet_create), and at a cold build without the stateful schedule; B200SQP_EINVAL on a
 *   centroidal handle (it has b200sqp_cen_set_motion_manager), for gait ids outside the builder table (at the call, or at the cold build for a
 *   table set later) and non-finite values.
 *   Builds with a manager: a non-finite cmd entry is B200SQP_EINVAL; on a cold build gait[b] must be one of the seven ids (the state starts at
 *   its row: the reference starts at stance) and t0 >= filter_origin, B200SQP_EINVAL otherwise; on a warm build gait is ignored and may be NULL
 *   (gait_start is checked as on every build and, as on every stateful warm build, not read).  A cold build evaluates no transition, whatever
 *   its t0: it seeds the state and the target buffer; the first transition can fire at the first warm build.
 *   b200sqp_download_motion_state: after a build with a manager, state [B] (0 stance .. 6 run), last_change [B] and filtered_cmd [B][4] of the
 *   last build, in caller order; any pointer may be NULL; B200SQP_ESTATE without such a build. */
typedef struct b200sqp_motion_desc {
  int32_t gait[7];                 /* builder gait ids of stance, slow_walk, walk, slower_trot, slow_trot, trot, run */
  double max_velocity_x;           /* reference.info maxDisplacementVelocityX */
  double max_velocity_y;           /* maxDisplacementVelocityY */
  double max_rotation_velocity;    /* maxRotationVelocity */
  double filter_origin;            /* the MPC time at which the command filter is constructed */
} b200sqp_motion_desc;
int b200sqp_set_motion_manager(b200sqp_handle h, const b200sqp_motion_desc* md);
/* The manager of the reference's centroidal MPC node (humanoid_centroidal_mpc_ros2 CentroidalMpcSqpNode.cpp:72-87, the configuration its launch
 * files start by default) on a centroidal handle, in the stateful mode of b200sqp_cen_set_gait_schedule; same descriptor, rules and error codes
 * as b200sqp_set_motion_manager, B200SQP_EINVAL on a whole-body handle.  Two things follow the centroidal model:
 *   - the targets are CentroidalMpcTargetTrajectoriesCalculator's (normalized momentum, base pose, default joints; see b200sqp_build_instances)
 *     of the filtered command, with the base velocity Ab^-1 hbar of the build's measured state, buffered with the same one-cycle delay;
 *   - the band transitions read getBaseComVelocity of the centroidal model, the normalized momentum hbar = x0[0 .. 6) itself
 *     (CentroidalMpcRobotModel.h:134-137), not Ab^-1 hbar; the "slower" test reads the command's |yaw rate| as on whole-body handles.
 * The scales are those of the centroidal reference.info (maxDisplacementVelocityX 2.4 there, 2.0 in the whole-body one).  The horizon of the
 * target rule is the build's horizon, where the reference passes mpcSettings.timeHorizon_: they agree when the build uses the task.info value. */
int b200sqp_cen_set_motion_manager(b200sqp_handle h, const b200sqp_motion_desc* md);
/* (on either family; in caller order on a fleet through b200sqp_fleet_download_motion_state) */
int b200sqp_download_motion_state(b200sqp_handle h, int32_t* state, double* last_change, double* filtered_cmd);

/* ------------------------------------------------------------------------------------------------------------------
 * Policy roll-out (SURVEY.md section 8(f)-2): MRT_BASE::rolloutPolicy (ocs2_mpc/src/MRT_BASE.cpp:124-151) of the reference's dummy
 * simulation, batched: TimeTriggeredRollout (ocs2_oc/src/rollout/TimeTriggeredRollout.cpp:46-116) with the OCP's whole-body flow map under the
 * policy of the last solve -- the LinearController u = bias(t) + K(t) x when settings.use_feedback_policy = 1, the FeedforwardController
 * otherwise -- integrated by the Dormand-Prince 5(4) stepper of ocs2 (ODE45_OCS2, ocs2_core/src/integration/RungeKuttaDormandPrince5.cpp).
 * The event times are the plan's PreEvent node times; the jump map is the identity.
 * ------------------------------------------------------------------------------------------------------------------ */
/* rollout::Settings fields of the ODE45 roll-out (ocs2_oc/include/ocs2_oc/rollout/RolloutSettings.h) */
typedef struct b200sqp_rollout_settings {
  double abs_tol, rel_tol;        /* AbsTolODE, RelTolODE */
  double time_step;               /* timeStep: initial step of every integration interval */
  double max_steps_per_second;    /* maxNumStepsPerSecond: flow-map call budget = this * max(1, duration) */
} b200sqp_rollout_settings;
/* the G1 whole-body task.info values: 1e-5, 1e-3, 0.015, 10000 */
void b200sqp_default_rollout_settings(b200sqp_rollout_settings* rs);

/* Simulates every instance from time t for `duration` seconds under the policy of the handle's last solve, ASYNCHRONOUS on `stream` like
 * b200sqp_solve (b200sqp_wait collects it; so does every entry point that waits for the handle).
 *   x_start [B][nx] host, or NULL for the handle's current measured state x0;
 *   outputs (host, each may be NULL, valid after b200sqp_wait): x_end [B][nx], u_end [B][nu] (the policy's input at the last sample),
 *   mode_end [B] (ModeSchedule::modeAtTime(t + duration): 0 FLY, 1 RF, 2 LF, 3 STANCE), n_steps [B][3] (accepted steps, rejected steps,
 *   flow-map calls), status [B] (0 ok; 1 more than 100 retries of one step; 2 the flow-map call budget was exceeded; 3 a non-finite state or
 *   input; the reference throws in these cases, here x_end holds the last accepted state).
 * The simulated state stays on the device as the handle's simulated measured state, which b200sqp_build_instances(warm = 2) takes as x0.
 * Like the reference, a t + duration past the plan's last node is not an error: the policy is held at its last node.
 * Needs a finished b200sqp_solve (B200SQP_ESTATE otherwise).  Whole-body handles only: a centroidal handle returns B200SQP_EINVAL here and
 * has its own entry point, b200sqp_cen_rollout_policy. */
int b200sqp_rollout_policy(b200sqp_handle h, double t, double duration, const double* x_start, const b200sqp_rollout_settings* rs, double* x_end,
                           double* u_end, int32_t* mode_end, int32_t* n_steps, int32_t* status, void* stream);

/* The policy roll-out of a centroidal handle (b200sqp_cen_create): CentroidalMpcDummySimNode.cpp:63-76 runs the MRT with
 * interface.getRollout(), a TimeTriggeredRollout over the OCP's own CentroidalDynamicsAD (CentroidalMpcInterface.cpp:107,231), so the flow map
 * is the handle's centroidal dynamics (either centroidalModelType).  Same parameters, outputs, errors and asynchrony as b200sqp_rollout_policy,
 * with x_start / x_end [B][12 + nj]; b200sqp_build_instances(warm = 2) takes its simulated state.  Whole-body handles: B200SQP_EINVAL.
 * The rollout block of the centroidal task.info (robot_models/unitree_g1/g1_centroidal_mpc/config/mpc/task.info:100-108) differs from the
 * whole-body one: AbsTolODE 5e-5, RelTolODE 5e-3, timeStep 0.015, maxNumStepsPerSecond 10000 (b200sqp_default_rollout_settings keeps the
 * whole-body values).  useFeedbackPolicy is false there, so the centroidal dummy loop runs the feed-forward controller by default, and its MRT
 * runs at 100 Hz against an 80 Hz MPC: one roll-out of 1/100 s per MPC cycle (MRT_ROS_Dummy_Loop.cpp:83). */
int b200sqp_cen_rollout_policy(b200sqp_handle h, double t, double duration, const double* x_start, const b200sqp_rollout_settings* rs, double* x_end,
                               double* u_end, int32_t* mode_end, int32_t* n_steps, int32_t* status, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * MRT joint controller (WBMpcMrtJointController / CentroidalMpcMrtJointController::computeJointControlAction), batched: the joint actions a
 * robot or a physics simulator consumes on every control tick, for whole-body and centroidal handles (the handle decides the family).
 *   robot_state [B][13 + 2 nj] host: one ::robot::model::RobotState per instance -- root position (world, 3), root orientation local-to-world
 *   as a quaternion in Eigen coefficient order x, y, z, w (4; used as given, not renormalised), root linear velocity (local frame, 3), root
 *   angular velocity (local frame, 3), joint positions and joint velocities in MPC joint order (nj each).  It is mapped into MPC coordinates as
 *   updateMpcState does: whole-body (position, quaternionToEulerZYX, joints, R v_local, Euler-ZYX rates, joint velocities); centroidal
 *   (hbar = A(q) v / m with the CMM of the handle's centroidalModelType, q).
 *   robot_state = NULL: the measured state is the end state of the handle's last roll-out, already in MPC coordinates (B200SQP_ESTATE without one).
 *   t: the time the policy is evaluated at.  Both reference controllers pass robotState.getTime() + 0.005; pass that.  A t past the plan's last
 *   node holds the last node, as in the reference.
 *   use_policy = 1 (initialPolicyReceived): the policy of the last finished b200sqp_solve (B200SQP_ESTATE without one), linear or feed-forward
 *   per settings.use_feedback_policy, evaluated at (t, x_obs); kp = 1200, kd = 10.
 *     whole-body: tau = computeJointTorques(x_policy, u_policy) (the map of b200sqp_joint_torques), q_des / qd_des = joint angles / velocities
 *     of x_policy, the planned state interpolated at t;
 *     centroidal: q_des = joint angles of x_policy, qd_des = joint velocities of u_policy, tau = computeJointTorques(q, qd, qdd_j = 0,
 *     wrenches of u_policy) at the MEASURED q, with qd = getGeneralizedVelocities(x_obs, 0) = (A_b^-1 m hbar, 0).  (The reference's
 *     inverse-dynamics PD gains are 0, so qdd_j = 0.)
 *   use_policy = 0 ("Apply weight compensating torque"; needs only a batch): u = weightCompensatingInput with both feet in stance, mode = 3,
 *   q_des = qd_des = 0; torques at the observation (whole-body) or at (q, qd) as above (centroidal).  kp / kd = 0 / 0 whole-body, 1200 / 10
 *   centroidal.
 *   Outputs (host, each may be NULL, valid after b200sqp_wait): q_des, qd_des, tau_ff [B][nj]; x_obs [B][nx] the observation; u_policy [B][nu];
 *   mode [B] (modeAtTime(t): 0 FLY, 1 RF, 2 LF, 3 STANCE).  Centroidal rows are 35 wide.
 * ASYNCHRONOUS on `stream` like b200sqp_rollout_policy.  The call reads the plan and the simulated state and writes neither: a later
 * b200sqp_build_instances(warm = 2) or roll-out behaves as if it had not been made.  The fixed (non-MPC) joints are the caller's: the
 * reference sends q_des = 0, kp = 100, kd = 1 and no torque for them.
 * B200SQP_EINVAL: null handle, non-finite t, use_policy not 0 or 1, a non-finite robot_state entry, or a quaternion whose norm is off 1 by more
 * than 1e-6. */
int b200sqp_joint_actions(b200sqp_handle h, double t, const double* robot_state, int use_policy, double* q_des, double* qd_des, double* tau_ff,
                          double* x_obs, double* u_policy, int32_t* mode, void* stream);

/* per-instance iteration record: mirrors sqp::LogEntry / PerformanceIndex (SqpLogging.h, PerformanceIndex.h) */
typedef struct b200sqp_iter_log {
  double base_merit, base_cost, base_dyn_sse, base_eq_sse;
  double merit, cost, dyn_sse, eq_sse;
  double step_size, step_type, dx_norm, du_norm, armijo, convergence;
  double pad[2];
} b200sqp_iter_log;

/* primalSolution / getRiccatiFeedback / getIterationsLog:
 *   x [B][n_nodes][nx], u [B][n_nodes-1][nu], K [B][n_nodes-1][nu*nx] (remapped gains, may be NULL),
 *   log [B][sqp_iteration] (rows from n_iter on are zeros), n_iter [B], status [B]: 0 ok; 1 QP failed (Cholesky of the projected input
 *   Hessian, NaN); 2 a whole-body constraint Jacobian D lost full row rank under Eigen::FullPivLU's threshold (the reference's
 *   luConstraintProjection would continue with a larger null space; this path reports it).  Any non-zero status makes the call return B200SQP_EQP. Synchronises. */
int b200sqp_download(b200sqp_handle h, double* x, double* u, double* K, b200sqp_iter_log* log, int32_t* n_iter, int32_t* status);

/* SqpSolver::getValueFunction data (needs settings.create_value_function): quadratic cost-to-go of the last iteration's QP,
 * re-centred on the linearisation trajectory as in extractValueFunction (dfdx -= dfdxx * x):  P [B][n_nodes][nx*nx], p [B][n_nodes][nx]. */
int b200sqp_download_value_function(b200sqp_handle h, double* P, double* p);

/* Centroidal flow map of the humanoid centroidal MPC (PinocchioCentroidalDynamicsAD::getValueCppAd,
 * lib/ocs2_ros2/ocs2_pinocchio/ocs2_centroidal_model/src/PinocchioCentroidalDynamicsAD.cpp:75-94) and its Jacobians
 * (SystemDynamicsBaseAD::linearApproximation), batched; the centroidal model shares the kinematic tree and contact frames of `model`.
 *   x [B][12+nj] = (normalized momentum 6, base position 3, Euler ZYX 3, joints nj); u [B][12+nj] = (wrench_l 6, wrench_r 6, joint velocities nj)
 *   xdot [B][12+nj]; dfdx [B][(12+nj)^2], dfdu [B][(12+nj)^2] column-major, either may be NULL.  Host pointers. */
int b200sqp_centroidal_flow_map(const b200sqp_model_desc* model, int batch, const double* x, const double* u, double* xdot, double* dfdx,
                                double* dfdu, int device);

/* ------------------------------------------------------------------------------------------------------------------
 * (3) Centroidal SQP solver: replaces ocs2::SqpSolver for the humanoid centroidal OCP
 *     (OCP wiring humanoid_nmpc/humanoid_centroidal_mpc/src/CentroidalMpcInterface.cpp:150-237; BASELINE configs 0-1).
 *     The handle is a b200sqp_handle: set_batch / upload_instances / reset / solve / download / download_value_function /
 *     download_stage_blocks / get_stage_times work on it unchanged, with nx = nu = 12 + nj in every array of the ABI
 *     (x = normalized momentum 6, base position 3, Euler ZYX 3, joints nj; u = wrench_l 6, wrench_r 6, joint velocities nj).
 *     `model` is filled from the centroidal task.info: Q_diag / R_diag / Qf_diag hold 12+nj entries, foot_cost_w[0..11] is
 *     EndEffectorKinematicsWeights::toVector() (position, orientation, linear velocity, angular velocity), foot_gain_pos_z / foot_gain_ori
 *     configure the stance twist and swing normal-velocity constraints, frame `torso_frame` of the frame table is the task-space link.
 *     swing_ref[..][2] (the swing-z acceleration) is ignored by this OCP.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_cen_desc {
  int32_t torso_frame;          /* index into model.frame_body / frame_p: link of the EndEffectorKinematicsQuadraticCost (task_space_costs) */
  double torso_R[9];            /* rotation of that link frame in its body's joint frame, row-major */
  double torso_w[12];           /* its EndEffectorKinematicsWeights */
  double icp_weight;            /* icp_cost_weights.icpErrorWeight */
  int32_t torque_joint[2][6];   /* ExternalTorqueQuadraticCostAD: active joints (0-based joint indices) per contact ... */
  double torque_w[2][6];        /* ... and their weights (left_leg_torque_cost / right_leg_torque_cost) */
  int32_t model_type;           /* centroidalModelType: 0 FullCentroidalDynamics, 1 SingleRigidBodyDynamics (CentroidalModelInfo.h:47) */
  double inertia_nominal[9];    /* SRBD only: CentroidalModelInfo::centroidalInertiaNominal (row-major) and comToBasePositionNominal, i.e. */
  double com_to_base_nominal[3];/* ccrba at q = (0_6, defaultJointState) (ocs2_centroidal_model/src/FactoryFunctions.cpp:113-121)          */
} b200sqp_cen_desc;
int b200sqp_cen_create(const b200sqp_model_desc* model, const b200sqp_cen_desc* cen, const b200sqp_settings* settings, int device,
                       b200sqp_handle* out);

/* Joint-torque map of the MRT controllers (computeJointTorques, humanoid_common_mpc/src/pinocchio_model/DynamicsHelperFunctions.cpp:232-270;
 * WBMpcMrtJointController.cpp:141): feed-forward torques of whole-body (x, u) samples, e.g. every node of a batch of primal solutions.
 *   x [count][2*(6+nj)], u [count][12+nj] -> tau [count][nj]; qddb [count][6] = the base acceleration of computeBaseAcceleration, may be NULL.
 * Host pointers; stateless. */
int b200sqp_joint_torques(const b200sqp_model_desc* model, int count, const double* x, const double* u, double* tau, double* qddb, int device);

/* Stage blocks of the last LQ approximation, for block-level parity tests:
 *   which = 0 raw (before projection): A [nx*nx] B [nx*nu] b [nx] Q S(nu x nx) R q r C(nc_max x nx) D(nc_max x nu) e nc
 *   see b200sqp_stage_layout for offsets. */
int b200sqp_download_stage_blocks(b200sqp_handle h, int which, double* out, int64_t out_doubles);
int b200sqp_stage_doubles(b200sqp_handle h, int which, int64_t* per_node);

/* SqpSolver::getBenchmarks(): device ms of {LQ approximation, solve QP, line search} of the last solve; ms[3] = the share of ms[0] spent in
 * the projection kernel (the reference's fourth timer, computeController, has no separate counterpart: the remap runs inside the QP stage) */
int b200sqp_get_stage_times(b200sqp_handle h, float ms[4]);
/* number of kernel launches issued by the last b200sqp_solve */
int b200sqp_get_launch_count(b200sqp_handle h, int64_t* launches);

/* ------------------------------------------------------------------------------------------------------------------
 * Fleets: the device-resident MPC loop for a batch whose instances differ in node count (different gait phases, different gaits, gait changes
 * at different cycles).  A fleet is attached to a handle (whole-body or centroidal) after b200sqp_set_builder and, optionally,
 * b200sqp_set_gait_schedule / b200sqp_set_motion_manager (b200sqp_cen_set_gait_schedule / b200sqp_cen_set_motion_manager on a centroidal handle),
 * and takes over its model, settings, builder and gait-schedule configuration and its device memory.  Every cycle the
 * builder's grid pass runs over all instances in caller order, a stable counting sort on the device groups them by node count (node count
 * ascending, caller order inside a group), and each group is solved as a view into the handle's batch allocation, one group after the other on
 * the caller's stream.  The regrouping never shows at the ABI: every array is in the caller's instance order, and the state carried from one
 * cycle to the next (the previous solution of warm = 1, x0 = NULL and warm = 2, the stateful gait schedule and its last command, the simulated
 * state of the last roll-out) follows each instance when it changes group.
 *   b200sqp_fleet_create: B200SQP_EINVAL with settings.global_step = 1; B200SQP_ESTATE without a builder or with a fleet already attached.
 *   While a fleet is attached, the handle's own compute entry points return B200SQP_ESTATE.  b200sqp_fleet_destroy detaches it; the handle
 *   then needs a cold build.  b200sqp_destroy destroys an attached fleet with its handle (the b200sqp_fleet is invalid afterwards).
 *   Before the fleet's first successful build, its solve, roll-out, joint-action and download entry points return B200SQP_ESTATE; so does a
 *   warm build whose horizon needs a larger batch allocation (the previous solutions live in it).
 *   b200sqp_fleet_build_instances: b200sqp_build_instances with per-instance node counts n_nodes [B] and *n_groups distinct counts; the warm
 *   semantics, call-order errors and messages are those of the handle (a new fleet has no previous solve: warm = 1 / 2 return B200SQP_ESTATE).
 *   b200sqp_fleet_solve / _wait / _rollout_policy / _joint_actions: as b200sqp_solve / b200sqp_wait / b200sqp_rollout_policy (on a centroidal
 *   handle b200sqp_cen_rollout_policy) / b200sqp_joint_actions, with the same arguments.
 *   b200sqp_fleet_download / _download_instances: the arrays of b200sqp_download / b200sqp_download_instances with max_nodes node rows per
 *   instance (max_nodes - 1 stage rows), the rows past an instance's n_nodes zero; B200SQP_EINVAL when an instance has more than max_nodes.
 *   b200sqp_fleet_get_stage_times: the stage times of b200sqp_get_stage_times summed over the groups of the last solve.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_fleet_t* b200sqp_fleet;
int b200sqp_fleet_create(b200sqp_handle h, b200sqp_fleet* out);
void b200sqp_fleet_destroy(b200sqp_fleet f);
int b200sqp_fleet_build_instances(b200sqp_fleet f, int batch, double t0, double horizon, const double* x0, const int32_t* gait, const double* gait_start,
                                  const double* cmd, int warm, int32_t* n_nodes, int32_t* n_groups);
int b200sqp_fleet_solve(b200sqp_fleet f, void* stream);
int b200sqp_fleet_wait(b200sqp_fleet f);
int b200sqp_fleet_rollout_policy(b200sqp_fleet f, double t, double duration, const double* x_start, const b200sqp_rollout_settings* rs, double* x_end,
                                 double* u_end, int32_t* mode_end, int32_t* n_steps, int32_t* status, void* stream);
int b200sqp_fleet_joint_actions(b200sqp_fleet f, double t, const double* robot_state, int use_policy, double* q_des, double* qd_des, double* tau_ff,
                                double* x_obs, double* u_policy, int32_t* mode, void* stream);
int b200sqp_fleet_download(b200sqp_fleet f, int max_nodes, double* x, double* u, double* K, b200sqp_iter_log* log, int32_t* n_iter, int32_t* status,
                           int32_t* n_nodes);
int b200sqp_fleet_download_instances(b200sqp_fleet f, int max_nodes, double* x0, double* x_init, double* u_init, double* t_nodes, uint8_t* node_event,
                                     uint8_t* contact_flags, double* swing_ref, double* impact_factor, double* arm_phase, double* x_ref, int32_t* n_nodes);
int b200sqp_fleet_download_mode_schedule(b200sqp_fleet f, int max_events, double* event_times, int32_t* mode_sequence, int32_t* n_events);
int b200sqp_fleet_get_stage_times(b200sqp_fleet f, float ms[4]);
/* b200sqp_download_motion_state of the fleet's instances (caller order) */
int b200sqp_fleet_download_motion_state(b200sqp_fleet f, int32_t* state, double* last_change, double* filtered_cmd);

/* ------------------------------------------------------------------------------------------------------------------
 * Per-instance resets: the episode loop of the reference's MpcnetRolloutBase (set: new observation, MPC reset, mode schedule and targets;
 * step: the episode ends when isValid fails) and the MPC reset service (MPC_BASE::reset, SqpSolver::reset), per instance on the device, so
 * that a failed or finished instance restarts without a cold build of the batch.  Needs the stateful gait schedule
 * (b200sqp_set_gait_schedule / b200sqp_cen_set_gait_schedule with stateful = 1): B200SQP_ESTATE otherwise (in the functional mode the caller
 * passes gait and gait_start every build, so there is no device schedule to restart).
 *   A reset of instance b at a warm build at time t0 starts a fresh episode whose clock starts at t0: b is built as a cold build would build
 *   it, with every time of that cold build shifted by t0.  x0[b] becomes the reset row (and so does the simulated state of b, so that
 *   b200sqp_joint_actions(robot_state = NULL) and the next roll-out start the new episode); the initial guess is the cold one (x_k = x0,
 *   WeightCompInitializer inputs), without warm shift or trajectorySpread; the gait schedule is fresh (the reset gait tiled from
 *   t0 + gait_offset, STANCE before it) and its command bookkeeping restarts at that gait (the caller's gait[b] of this one build is ignored);
 *   a motion manager restarts at the row of the reset gait with its last change and its filter's origin at t0, and takes this build's cmd[b]
 *   for its targets.  Every other instance gets the warm build it would have had without resets, bit for bit.  A cold build starts every
 *   instance in episode 0 at its t0 and drops pending requests.
 *   On a plain handle a reset that changes the node count fails with the "between %d and %d shooting nodes" B200SQP_EINVAL of
 *   b200sqp_build_instances, after which the next build must be cold (as after every failed stateful warm build); fleets have no such limit.
 *   When reset states were never set, builds run exactly as before and launch nothing more.
 * b200sqp_set_reset_states: reset rows of `batch` instances: x0 [B][nx] (12 + nj on centroidal handles), gait [B] (builder table; one of the
 *   manager's seven when a manager is set), gait_offset [B] <= 0.5 (tiling starts at t0 + offset).  Stored on the device; may be replaced at
 *   any time.  B200SQP_EINVAL: a non-finite row entry, a gait id outside the table, an offset > 0.5, or a batch other than the built one (a
 *   build of another batch size also returns B200SQP_EINVAL while they are set).
 * b200sqp_set_auto_reset: the automatic predicate, evaluated per instance at the start of each warm build, first matching reason recorded:
 *   non-finite measured state (always); last solve status != 0 (on_solve_failure); last roll-out status != 0 (on_rollout_failure, warm = 2
 *   builds only); |height - height_reset|, |pitch - pitch_reset|, |roll - roll_reset| above its bound (the reference values from the
 *   instance's reset row, as isValid compares with the default state; whole-body x[2], x[4], x[5], centroidal x[8], x[10], x[11]).  A bound
 *   of 0 switches that test off; negative or non-finite bounds: B200SQP_EINVAL.  NULL: off.  Set it on the handle before b200sqp_fleet_create.
 *   Takes effect once reset states are set.
 * b200sqp_request_resets: the given instances are reset at the next warm build (reason 1, ahead of the predicate).  B200SQP_EINVAL for an
 *   index outside [0, B); B200SQP_ESTATE without reset states.
 * b200sqp_download_episodes: after a build, per instance: episode [B] (0 from the cold build on), episode_start [B] (t0 of the episode's
 *   first build), reason [B] (0 not reset at the last build, 1 requested, 2 non-finite, 3 solve, 4 roll-out, 5 height, 6 pitch, 7 roll),
 *   reset [B] (1: reset at the last build), last_length [B] (t0 - start of the episode that the last reset ended: the reference's
 *   survivalTime); any pointer may be NULL.  B200SQP_ESTATE without reset states.
 * The handle entry points return B200SQP_ESTATE while a fleet is attached; the fleet's take the same arguments in caller order.
 * ------------------------------------------------------------------------------------------------------------------ */
int b200sqp_set_reset_states(b200sqp_handle h, int batch, const double* x0, const int32_t* gait, const double* gait_offset);
typedef struct b200sqp_auto_reset_desc {
  int32_t on_solve_failure, on_rollout_failure;
  double max_height_deviation, max_pitch_deviation, max_roll_deviation;   /* 0: that test off */
} b200sqp_auto_reset_desc;
int b200sqp_set_auto_reset(b200sqp_handle h, const b200sqp_auto_reset_desc* d);
int b200sqp_request_resets(b200sqp_handle h, int count, const int32_t* instances);
int b200sqp_download_episodes(b200sqp_handle h, int32_t* episode, double* episode_start, int32_t* reason, uint8_t* reset, double* last_length);
int b200sqp_fleet_set_reset_states(b200sqp_fleet f, int batch, const double* x0, const int32_t* gait, const double* gait_offset);
int b200sqp_fleet_request_resets(b200sqp_fleet f, int count, const int32_t* instances);
int b200sqp_fleet_download_episodes(b200sqp_fleet f, int32_t* episode, double* episode_start, int32_t* reason, uint8_t* reset, double* last_length);

/* ------------------------------------------------------------------------------------------------------------------
 * Pose commands: the reference's commandedPositionToTargetTrajectories (WBMpcPoseCommandNode, CentroidalMpcKeyboardPoseCommandNode) per
 * instance on the device, for whole-body and centroidal handles.  A command delta = (dx, dy, dz, dyaw) -- dx, dy in the pelvis frame, dz the
 * pelvis height offset from default_base_height, dyaw in degrees -- is latched from the instance's measured state x0 at t0 of the next build
 * (cold or warm, whichever source x0 came from: the caller, the previous plan, or the last roll-out):
 *   current = base pose of x0 (whole-body x[0..6), centroidal x[6..12), ZYX Euler) with pitch and roll 0;
 *   target  = (current[0..2) + (dx, dy) rotated by current yaw, default_base_height + clamp(dz, +-max_delta_pelvis_height),
 *              current yaw + dyaw * pi / 180, 0, 0);
 *   t_reach = t0 + max(|target yaw - current yaw| / target_rotation_velocity, |(target - current)[0..2)| / target_displacement_velocity);
 *   knots {t0: current, t_reach: target}, whole-body [pose, default joints, 0], centroidal [0_6, pose, default joints], interpolated
 *   linearly and clamped at both ends (t_reach = t0: the target at every node after t0).
 * The latched target stays fixed in the world frame over the following builds, in place of the velocity command, until it is cleared
 * (b200sqp_clear_poses: the velocity rule again from the next build), re-latched by a new command, dropped by a reset of the instance
 * (b200sqp_request_resets or the automatic predicate), or dropped by a cold build (which drops every target first, then latches the
 * commands pending for it).  A second command before a build replaces the first.
 * b200sqp_set_pose_commands: enables pose commands (pd != NULL) with the reference.info values, or disables them (NULL: every instance
 *   follows its velocity command again from the next build).  B200SQP_EINVAL for a non-positive or non-finite speed, a negative or
 *   non-finite max_delta_pelvis_height or a non-finite default_base_height; B200SQP_ESTATE with a motion manager set (the manager
 *   rewrites the targets every cycle; b200sqp_set_motion_manager returns B200SQP_ESTATE while pose commands are on).
 * b200sqp_command_poses / b200sqp_clear_poses: instances [count] of the built batch, delta [count][4].  B200SQP_EINVAL for an index
 *   outside [0, B) or a non-finite delta; B200SQP_ESTATE before b200sqp_set_pose_commands, with a motion manager, or before the first build.
 *   Commands pending when the batch size changes are dropped.
 * b200sqp_download_pose_targets: per instance after a build: active [B] (1: the pose targets were used), t_start [B], t_reach [B],
 *   target_pose [B][6], error [B][2] (planar distance and |yaw - target yaw| of that build's measured state; 0 when not active); any
 *   pointer may be NULL.  B200SQP_ESTATE when nothing was built with pose commands on.
 * When pose commands were never enabled, builds launch nothing more and compute exactly what they computed before.  The handle entry
 * points return B200SQP_ESTATE while a fleet is attached (set_pose_commands on the handle before b200sqp_fleet_create); the fleet's take
 * the same arguments in caller order.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_pose_desc {
  double target_displacement_velocity;   /* reference.info targetDisplacementVelocity (> 0) */
  double target_rotation_velocity;       /* targetRotationVelocity (> 0) */
  double max_delta_pelvis_height;        /* maxDeltaPelvisHeight (>= 0) */
  double default_base_height;            /* defaultBaseHeight */
} b200sqp_pose_desc;
int b200sqp_set_pose_commands(b200sqp_handle h, const b200sqp_pose_desc* pd);
int b200sqp_command_poses(b200sqp_handle h, int count, const int32_t* instances, const double* delta);
int b200sqp_clear_poses(b200sqp_handle h, int count, const int32_t* instances);
int b200sqp_download_pose_targets(b200sqp_handle h, int32_t* active, double* t_start, double* t_reach, double* target_pose, double* error);
int b200sqp_fleet_command_poses(b200sqp_fleet f, int count, const int32_t* instances, const double* delta);
int b200sqp_fleet_clear_poses(b200sqp_fleet f, int count, const int32_t* instances);
int b200sqp_fleet_download_pose_targets(b200sqp_fleet f, int32_t* active, double* t_start, double* t_reach, double* target_pose, double* error);

/* ------------------------------------------------------------------------------------------------------------------
 * Device-pointer I/O: the boundary of the closed loop in GPU memory, for a batched simulator whose robot states already live on the device.
 * Every pointer argument below is device (or managed) memory on the handle's device, except gait, gait_start, cmd, n_nodes and n_groups,
 * which are host arrays as in the host entry points.  Each device pointer is checked with cudaPointerGetAttributes: anything else returns
 * B200SQP_EINVAL and enqueues nothing.  `stream` is a cudaStream_t (NULL: the legacy default stream).
 *
 * b200sqp_build_instances_dev / b200sqp_fleet_build_instances_dev: b200sqp_build_instances / b200sqp_fleet_build_instances with the measured
 *   states x0_dev [B][nx] (35 wide on centroidal handles) in device memory; x0_dev is required (x0 = NULL builds use the host entry points)
 *   and warm is 0 or 1 (warm = 2 takes the simulated state: B200SQP_EINVAL).  The build reads x0_dev after the work enqueued on `stream`
 *   before the call (a producer kernel of the caller is seen).  Everything else, synchronisation and return codes included, is the host build.
 * b200sqp_joint_actions_dev / b200sqp_fleet_joint_actions_dev: b200sqp_joint_actions with robot_state_dev [B][13 + 2 nj] in device memory
 *   (NULL: the end state of the last roll-out) and every output in device memory (each may be NULL).  The call enqueues its work on `stream`
 *   and returns: no host synchronisation, no pageable copy, no allocation after the first call at a batch size.  The robot-state check of
 *   the host entry point (every entry finite, |quaternion norm - 1| <= 1e-6) runs on the device per row and writes status [B] (may be NULL):
 *   0 accepted, 1 an entry is not finite, 2 the quaternion norm is off.  A rejected row gets NaN in every double output and mode -1; every
 *   other row is bit-identical to what b200sqp_joint_actions returns for it.  B200SQP_EINVAL (t, use_policy) and B200SQP_ESTATE (no batch,
 *   solve or roll-out) as on the host path.
 * b200sqp_download_dev / b200sqp_fleet_download_dev: the x, u, K and status outputs of b200sqp_download / b200sqp_fleet_download (caller order,
 *   fleets padded to max_nodes rows with zeros, centroidal rows 35 wide), enqueued on `stream`; each may be NULL.  status [B] is the
 *   per-instance solve status: the call cannot see it without a synchronisation, so it returns 0 where the host download returns
 *   B200SQP_EQP.  K needs settings.use_feedback_policy (B200SQP_ESTATE).  n_nodes [B] (fleet, host, may be NULL): each instance's node count.
 *
 * Ordering: calls on one handle run on the device in the order they were made, whatever streams they are given.  A _dev call enqueues behind
 *   the handle's outstanding work (a solve or roll-out in flight, the last _dev call) with stream waits, not host waits, and records an event
 *   after its own work; every entry point that touches what a _dev call reads or writes (the plan, the simulated state, the joint-action
 *   scratch, the fleet carry) makes its stream wait on that event before it enqueues anything, and memory is not freed under it.
 *   b200sqp_wait / b200sqp_fleet_wait also wait for outstanding _dev work.  When no _dev call was made, nothing new is recorded or waited on.
 * ------------------------------------------------------------------------------------------------------------------ */
int b200sqp_build_instances_dev(b200sqp_handle h, int batch, double t0, double horizon, const double* x0_dev, const int32_t* gait,
                                const double* gait_start, const double* cmd, int warm, int32_t* n_nodes, void* stream);
int b200sqp_fleet_build_instances_dev(b200sqp_fleet f, int batch, double t0, double horizon, const double* x0_dev, const int32_t* gait,
                                      const double* gait_start, const double* cmd, int warm, int32_t* n_nodes, int32_t* n_groups, void* stream);
int b200sqp_joint_actions_dev(b200sqp_handle h, double t, const double* robot_state_dev, int use_policy, double* q_des, double* qd_des, double* tau_ff,
                              double* x_obs, double* u_policy, int32_t* mode, int32_t* status, void* stream);
int b200sqp_fleet_joint_actions_dev(b200sqp_fleet f, double t, const double* robot_state_dev, int use_policy, double* q_des, double* qd_des,
                                    double* tau_ff, double* x_obs, double* u_policy, int32_t* mode, int32_t* status, void* stream);
int b200sqp_download_dev(b200sqp_handle h, double* x, double* u, double* K, int32_t* status, void* stream);
int b200sqp_fleet_download_dev(b200sqp_fleet f, int max_nodes, double* x, double* u, double* K, int32_t* status, int32_t* n_nodes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * MRT-side queries of the last solve: MPC_MRT_Interface::getValueFunction(time, state) (= SqpSolver::getValueFunction, SqpSolver.cpp:172-191)
 * and getLinearFeedbackGain(time) (LinearController::getFeedbackGain), batched, at one time t shared by every instance.  Per instance b, on its
 * own plan (its own node count on a fleet):
 *   (idx, alpha) = LinearInterpolation::timeSegment(t_nodes[b], t): t before the first node holds the first node, t past the last node the
 *   last, and a segment not longer than 2 weakEpsilon (a PreEvent / PostEvent pair) snaps to its nearer end;
 *   vf_dfdxx [B][nx*nx] = alpha P[idx] + (1 - alpha) P[idx + 1] entry-wise (column-major), P as b200sqp_download_value_function returns it;
 *   vf_dfdx [B][nx]     = alpha p[idx] + (1 - alpha) p[idx + 1], then dfdx_r += dfdxx_rc x_c for c = 0 .. nx-1 in that order (the re-centring
 *                         at x); the constant f is not produced (the reference sets it to 0);
 *   K [B][nu*nx]        = alpha K_src(idx) + (1 - alpha) K_src(idx + 1) entry-wise (column-major), src the stage whose gain node k carries
 *                         (toPrimalSolution: PreEvent nodes and the terminal node take the stage before them) -- the gain the linear policy of
 *                         b200sqp_rollout_policy / b200sqp_joint_actions uses at t.
 *   Every product and sum is rounded on its own, in the order above, so the results equal that formula on the host bit for bit.
 *   x [B][nx]: the state dfdx is re-centred at, read only when vf_dfdx is wanted; NULL: the end state of the last roll-out (as
 *   b200sqp_joint_actions(robot_state = NULL)).  Centroidal handles: nx = nu = 35 (the leading 35 rows and columns of the device blocks).
 *   Outputs: each may be NULL; with all three NULL the call returns 0 and enqueues nothing.  Caller order on fleets.
 * b200sqp_mrt_query / b200sqp_fleet_mrt_query: host arrays, ASYNCHRONOUS on `stream` like b200sqp_joint_actions (x is copied before the call
 *   returns; the outputs are valid after b200sqp_wait / b200sqp_fleet_wait).
 * b200sqp_mrt_query_dev / b200sqp_fleet_mrt_query_dev: x and every output in device memory, under the rules of the device-pointer I/O section
 *   (pointer check, stream waits, event after the call's work).
 * The query reads the plan, the cost-to-go, the gains and the simulated state and writes none of them: a later build, roll-out, joint-action
 * call or solve behaves as if it had not been made.
 * B200SQP_EINVAL: null handle, non-finite t, a _dev pointer that is not device memory.  B200SQP_ESTATE: nothing solved yet (a fleet before its
 * first build); vf_dfdxx or vf_dfdx with settings.create_value_function = 0; K with settings.use_feedback_policy = 0 (a feed-forward policy, where
 * the reference throws); x = NULL with vf_dfdx and no roll-out of the batch.  The handle entry points return B200SQP_ESTATE while a fleet is
 * attached.
 * b200sqp_fleet_download_value_function: b200sqp_download_value_function of a fleet, in caller order with max_nodes node rows per instance
 *   (the rows past n_nodes[b] zero): P [B][max_nodes][nx*nx], p [B][max_nodes][nx], n_nodes [B] (may be NULL).  Synchronises.
 *   B200SQP_EINVAL for a null P or p or an instance with more than max_nodes nodes; B200SQP_ESTATE as b200sqp_download_value_function.
 * ------------------------------------------------------------------------------------------------------------------ */
int b200sqp_mrt_query(b200sqp_handle h, double t, const double* x, double* vf_dfdxx, double* vf_dfdx, double* K, void* stream);
int b200sqp_fleet_mrt_query(b200sqp_fleet f, double t, const double* x, double* vf_dfdxx, double* vf_dfdx, double* K, void* stream);
int b200sqp_mrt_query_dev(b200sqp_handle h, double t, const double* x, double* vf_dfdxx, double* vf_dfdx, double* K, void* stream);
int b200sqp_fleet_mrt_query_dev(b200sqp_fleet f, double t, const double* x, double* vf_dfdxx, double* vf_dfdx, double* K, void* stream);
int b200sqp_fleet_download_value_function(b200sqp_fleet f, int max_nodes, double* P, double* p, int32_t* n_nodes);

/* ------------------------------------------------------------------------------------------------------------------
 * Per-instance gains: the reference's GainsReceiver (humanoid_centroidal_mpc_ros2 src/gains/GainsReceiver.cpp), a synchronized module whose
 * preSolverRun writes the newest gains message into the OCP's cost and soft-constraint terms, per instance of the batch on the device.
 * A gain set belongs to one instance index of the built batch (caller order, also on a fleet) and takes effect at that instance's next solve,
 * stream-ordered behind the work already enqueued on the handle.  Gains persist across solves, warm and cold builds of the same batch size and
 * per-instance resets; they are dropped (every instance back to the model's values) when the batch size changes, or for the listed instances
 * by b200sqp_set_gains(..., gains = NULL).  An inactive term (*_active = 0) contributes exactly zero to value, gradient and Hessian of that
 * instance (its weights, or its penalty's mu, are zero in the instance's model); its stored values come back when it is turned on again.
 * Gains change the OCP only: the policy roll-outs, the joint-action controller and the builder read the handle's model.  Not tunable: the
 * equality constraints (switching one off changes the projection sizes), the ICP and external-torque costs, fric_coeff and foot_gain_*.
 * When gains were never set, solves launch nothing more and compute exactly what they computed before.
 * b200sqp_default_gains: the handle's model values, every term active.
 * b200sqp_set_gains: count records for instances [count] (distinct, in [0, B)); gains = NULL restores the model's values.  Every used weight
 *   must be finite and >= 0, R_diag entries > 0 (the Riccati recursion factorises R~), mu >= 0, delta > 0, radii >= 0, flags 0 or 1:
 *   B200SQP_EINVAL otherwise, and nothing is applied.  Synchronous like the other host entry points.
 * b200sqp_download_gains: every instance's current record gains [B] (each may be NULL) and custom [B] (1: set by b200sqp_set_gains).
 * b200sqp_set_gains_dev: b200sqp_set_gains with the records in device memory (instances on the host), enqueued on `stream` under the
 *   ordering rules of the device-pointer I/O section.  The checks run on the device per row: status_dev [count] (may be NULL) gets 0 applied,
 *   1 an entry is not finite, 2 an entry is out of range; a rejected row leaves its instance unchanged.  The first set_gains call at a batch
 *   size (either path) allocates the per-instance models and waits for the handle's outstanding work; later calls do neither.
 * B200SQP_ESTATE before a batch exists (b200sqp_set_batch or a build), and on the handle entry points while a fleet is attached.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_gains {
  double Q_diag[64], R_diag[48], Qf_diag[64];  /* nx / nu entries used: 58 / 35 whole-body, 35 / 35 centroidal */
  double foot_cost_w[18];                      /* whole-body: EndEffectorDynamicsWeights (18); centroidal: the feet's EndEffectorKinematicsWeights (12) */
  double torso_w[12];                          /* centroidal: the task-space link's EndEffectorKinematicsWeights; ignored on whole-body handles */
  double jlim_mu, jlim_delta;                  /* JointLimitsSoftConstraint */
  double coll_mu, coll_delta, coll_r_foot, coll_r_knee;  /* FootCollisionConstraint and its sphere radii */
  double fric_mu, fric_delta;                  /* FrictionForceConeConstraint relaxed barrier */
  double momxy_mu, momxy_delta;                /* ContactMomentXY relaxed barrier */
  int32_t final_cost_active, foot_cost_active, torso_cost_active, joint_limits_active,
          foot_collision_active, friction_cone_active, contact_moment_active;
} b200sqp_gains;
int b200sqp_default_gains(b200sqp_handle h, b200sqp_gains* out);
int b200sqp_set_gains(b200sqp_handle h, int count, const int32_t* instances, const b200sqp_gains* gains /* [count] or NULL */);
int b200sqp_download_gains(b200sqp_handle h, b200sqp_gains* gains /* [B] */, int32_t* custom /* [B] */);
int b200sqp_set_gains_dev(b200sqp_handle h, int count, const int32_t* instances, const b200sqp_gains* gains_dev, int32_t* status_dev, void* stream);
int b200sqp_fleet_set_gains(b200sqp_fleet f, int count, const int32_t* instances, const b200sqp_gains* gains);
int b200sqp_fleet_download_gains(b200sqp_fleet f, b200sqp_gains* gains, int32_t* custom);
int b200sqp_fleet_set_gains_dev(b200sqp_fleet f, int count, const int32_t* instances, const b200sqp_gains* gains_dev, int32_t* status_dev,
                                void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Per-instance robot parameters: the link masses, centres of mass and inertias of one instance, for two targets.
 *   B200SQP_PARAMS_MODEL: what the instance's controller believes: the OCP (LQ approximation and line-search roll-out), the builder's
 *     weight-compensating inputs, centroidal target rule and base velocity, and the joint-action controller (b200sqp_joint_actions).  The
 *     builder weighs the instance with the record's sequential sum of the link masses in place of b200sqp_builder_desc.total_mass, unless
 *     the record's masses are the handle's.  (A total_mass set away from the sum of the description's link masses is thus replaced, not
 *     offset, for an instance whose record changes a link mass.)
 *   B200SQP_PARAMS_PLANT: what the instance's dummy simulation integrates: b200sqp_rollout_policy / b200sqp_cen_rollout_policy and the
 *     fleet's roll-out.  The plant is the same flow map with these inertial parameters.
 * The kinematic tree, joint frames, operational frames, contact geometry, joint limits and fric_coeff stay the handle's.  A record belongs to
 * one instance index of the built batch (caller order, also on a fleet) and takes effect at that instance's next build, solve, roll-out or
 * joint-action call, stream-ordered.  Records persist across solves, warm and cold builds of the same batch size and resets; they are dropped
 * when the batch size changes.  Gains (b200sqp_set_gains) and parameters compose: an instance's model is the handle's, then its model record,
 * then its gains, whichever was set first.  When no record was ever set, nothing more is launched or read.
 * b200sqp_default_robot_params: the handle's values (inertia_nominal / com_to_base_nominal those of its b200sqp_cen_desc on SRBD handles, else 0).
 * b200sqp_set_robot_params: count records for instances [count] (distinct, in [0, B)) and the targets `which` (a mask of the two flags);
 *   p = NULL restores the handle's values.  Every used entry (bodies 0..nj) must be finite, every mass >= 0 and their sum > 0, and every
 *   inertia (and inertia_nominal on SRBD handles) symmetric to 1e-12 relative and positive semi-definite (principal minors >= 0, to the same
 *   tolerance): B200SQP_EINVAL otherwise, and nothing is applied.  Synchronous.
 * b200sqp_download_robot_params: the current records of target `which` (1 or 2), p [B] and custom [B] (1: set), each may be NULL.
 * b200sqp_set_robot_params_dev: the records in device memory, enqueued on `stream` under the ordering rules of the device-pointer I/O
 *   section; status_dev [count] (may be NULL): 0 applied, 1 an entry is not finite, 2 an entry is out of range (a rejected row changes nothing).
 * The first call at a batch size (either path) allocates the per-instance models and waits for the handle's outstanding work; later calls do
 * neither.  B200SQP_ESTATE before a batch exists, and on the handle entry points while a fleet is attached.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct b200sqp_robot_params {
  double mass[B200SQP_MAX_BODIES];        /* per body, nj + 1 used (body 0 = floating base), as b200sqp_model_desc.mass */
  double com[B200SQP_MAX_BODIES][3];      /* as b200sqp_model_desc.com (body frame) */
  double inertia[B200SQP_MAX_BODIES][9];  /* as b200sqp_model_desc.inertia (about the com, row-major) */
  double inertia_nominal[9];              /* SRBD centroidal handles only: b200sqp_cen_desc.inertia_nominal ... */
  double com_to_base_nominal[3];          /* ... and com_to_base_nominal for these masses; ignored elsewhere */
} b200sqp_robot_params;
#define B200SQP_PARAMS_MODEL 1
#define B200SQP_PARAMS_PLANT 2
int b200sqp_default_robot_params(b200sqp_handle h, b200sqp_robot_params* out);
int b200sqp_set_robot_params(b200sqp_handle h, int count, const int32_t* instances, const b200sqp_robot_params* p /* [count] or NULL */,
                             int which);
int b200sqp_download_robot_params(b200sqp_handle h, int which, b200sqp_robot_params* p /* [B] */, int32_t* custom /* [B] */);
int b200sqp_set_robot_params_dev(b200sqp_handle h, int count, const int32_t* instances, const b200sqp_robot_params* p_dev, int which,
                                 int32_t* status_dev, void* stream);
int b200sqp_fleet_set_robot_params(b200sqp_fleet f, int count, const int32_t* instances, const b200sqp_robot_params* p, int which);
int b200sqp_fleet_download_robot_params(b200sqp_fleet f, int which, b200sqp_robot_params* p, int32_t* custom);
int b200sqp_fleet_set_robot_params_dev(b200sqp_fleet f, int count, const int32_t* instances, const b200sqp_robot_params* p_dev, int which,
                                       int32_t* status_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SQP_H */
