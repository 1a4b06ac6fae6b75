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

/* HpipmInterface::HpipmInterface(OcpSize) / resize(): allocate device storage for `batch` problems of N stages. */
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

/* SqpSolver::SqpSolver(settings, ocp, initializer) */
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
 * instance needs at most ceil(log(alpha_min) / log(alpha_decay)) + 1 trials, all of them are enqueued, and the thread blocks of an instance
 * whose search has ended return at their first instruction (likewise every kernel for a converged instance).  b200sqp_wait -- or any entry
 * point that reads results or re-uses the handle (download*, get_stage_times, reset, upload / build_instances, set_batch, destroy) -- waits for
 * the stream first.  One solve per handle in flight; several handles on several streams overlap on the device.  (The global-step mode takes a
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
 * walks the fixed ladder alpha_j = alpha_decay^j >= alpha_min from the largest candidate: one roll-out of every active instance, the
 * reference's filter test (FilterLinesearch.cpp:34-57), and
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
 * a warm build after a failed stateful warm build (its schedules were already advanced).  Centroidal handles, negative or non-finite times: B200SQP_EINVAL. */
int b200sqp_set_gait_schedule(b200sqp_handle h, int stateful, double phase_transition_stance_time);

/* The window mode schedule [t0 - T, tf + T] the last b200sqp_build_instances used, in either mode: event_times [B][max_events],
 * mode_sequence [B][max_events + 1] (modes after the n_events[b] + 1 used entries are -1), n_events [B].  B200SQP_EINVAL when an instance has
 * more than max_events events. */
int b200sqp_download_mode_schedule(b200sqp_handle h, int max_events, double* event_times, int32_t* mode_sequence, int32_t* n_events);

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

/* per-instance iteration record: mirrors sqp::LogEntry / PerformanceIndex (SqpLogging.h, PerformanceIndex.h) */
typedef struct b200sqp_iter_log {
  double base_merit, base_cost, base_dyn_sse, base_eq_sse;
  double merit, cost, dyn_sse, eq_sse;
  double step_size, step_type, dx_norm, du_norm, armijo, convergence;
  double pad[2];
} b200sqp_iter_log;

/* primalSolution / getRiccatiFeedback / getIterationsLog:
 *   x [B][n_nodes][nx], u [B][n_nodes-1][nu], K [B][n_nodes-1][nu*nx] (remapped gains, may be NULL),
 *   log [B][sqp_iteration], n_iter [B], status [B]: 0 ok; 1 QP failed (Cholesky of the projected input Hessian, NaN); 2 a whole-body
 *   constraint Jacobian D lost full row rank under Eigen::FullPivLU's threshold (the reference's luConstraintProjection would continue with a
 *   larger null space; this path reports it).  Any non-zero status makes the call return B200SQP_EQP. Synchronises. */
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

#ifdef __cplusplus
}
#endif
#endif /* B200SQP_H */
