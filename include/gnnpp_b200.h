/*
 * gnnpp_b200.h -- C ABI of libgnnpp_b200.so: the H100 (sm_90a) implementation of the
 * DecentralPlannerNet forward path of proroklab/gnn_pathplanning.
 *
 * The reference has no FFI of its own: its boundary for this path is the PyTorch
 * nn.Module API (SURVEY.md section 8b).  This header is the C-level boundary a
 * reference maintainer binds to (ctypes stub in INTEGRATION.md); every entry point
 * names the reference code it replaces.  Plain pointers and sizes only -- no torch
 * types.  All functions return 0 on success, a negative gpp_status otherwise;
 * gpp_last_error() returns a thread-local human-readable message.
 *
 * Conventions
 *   B batch (episodes), N agents (graph nodes), G input / F output features,
 *   K filter taps, E = 1 edge feature (the only value the reference path constructs,
 *   graphs/models/decentralplanner.py:209).
 *   `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   "dev" pointers are device memory, "host" pointers are host memory (pinned for
 *   full copy speed); neither is retained after the call returns unless stated.
 */
#ifndef GNNPP_B200_H
#define GNNPP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum gpp_status {
    GPP_OK = 0,
    GPP_ERR_INVALID = -1,     /* bad argument / shape (the reference raises AssertionError) */
    GPP_ERR_UNSUPPORTED = -2, /* valid in the reference but outside this library's envelope */
    GPP_ERR_CUDA = -3,        /* CUDA runtime error (message has the cudaError string) */
    GPP_ERR_NODEVICE = -4     /* no sm_90 device visible */
} gpp_status;

/* Tensor layouts of the node-signal tensors x / y. */
typedef enum gpp_layout {
    GPP_FEATURE_MAJOR = 0, /* [B, G, N]: the reference API layout (graphML.py:2298-2306) */
    GPP_NODE_MAJOR = 1     /* [B, N, G]: the native layout between the fused stages */
} gpp_layout;

const char* gpp_last_error(void);
int gpp_abi_version(void);
/* Fills SM count and compute capability of the current device. */
int gpp_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------
 * Graph filter  (replaces BatchLSIGF, utils/graphUtils/graphML.py:2273-2367, as called
 * by GraphFilterBatch.forward :2458-2477)
 *
 *   z_0 = x ; z_k = z_{k-1} . S_b  (right multiplication, :2350)
 *   y[b,f,n] = sum_{k,g} w[f,0,k,g] z_k[b,g,n] + bias[f]          (:2361-2366)
 *
 *   x      dev f32, layout x_layout, B*G*N
 *   S      dev [B,N,N], f32 or (s_is_f64 != 0) f64 -- cast to f32 per element exactly as
 *          `S.float()` does at :2350
 *   w      dev f32 [F,1,K,G]  (the module's `weight`, untouched layout)
 *   bias   dev f32 [F] or NULL
 *   y      dev f32, layout y_layout, B*F*N
 *   fuse_relu  apply max(.,0) in the epilogue (the nn.ReLU that follows the filter in
 *          DecentralPlannerNet.GFL, decentralplanner.py:221)
 *   workspace  dev scratch of gpp_graph_filter_workspace_bytes() bytes (holds the
 *          k-major transposed taps); may be NULL only if that size is 0
 * ---------------------------------------------------------------------------------- */
size_t gpp_graph_filter_workspace_bytes(int G, int F, int K);

int gpp_graph_filter_forward(const float* x, const void* S, int s_is_f64,
                             const float* w, const float* bias, float* y,
                             int B, int N, int G, int F, int K,
                             int x_layout, int y_layout, int fuse_relu,
                             void* workspace, void* stream);

/* Backward of the same filter (replaces autograd through graphML.py:2342-2366).
 *   dy   dev f32 [B,F,N]/[B,N,F] (y_layout) upstream gradient
 *   y    dev f32, the forward OUTPUT (needed only when fuse_relu, for the mask), else NULL
 *   dx   dev f32 out, x_layout         (NULL to skip)
 *   dw   dev f32 out [F,1,K,G]         (NULL to skip; overwritten, not accumulated)
 *   dbias dev f32 out [F]              (NULL to skip; overwritten)
 *   workspace: gpp_graph_filter_backward_workspace_bytes() bytes of dev scratch.
 * S receives no gradient (the reference's GSO never requires grad). */
size_t gpp_graph_filter_backward_workspace_bytes(int B, int N, int G, int F, int K);

int gpp_graph_filter_backward(const float* dy, const float* y, const float* x,
                              const void* S, int s_is_f64, const float* w,
                              float* dx, float* dw, float* dbias,
                              int B, int N, int G, int F, int K,
                              int x_layout, int y_layout, int fuse_relu,
                              void* workspace, void* stream);

/* ------------------------------------------------------------------------------------
 * Whole-planner inference  (replaces DecentralPlannerNet.addGSO + forward in eval mode,
 * graphs/models/decentralplanner.py:266-318: per-agent CNN + compress MLP -> K-tap graph
 * filter + ReLU -> per-agent action MLP)
 * ---------------------------------------------------------------------------------- */
typedef struct gpp_planner gpp_planner;

/* All pointers use the reference's state_dict shapes (SURVEY.md section 8 a1):
 *   conv_w[l]  [C_{l+1}, C_l, 3, 3]   conv_b[l] [C_{l+1}]     C = 3,32,32,64,64,128
 *   bn_w/bn_b/bn_mean/bn_var[l] [C_{l+1}]   (eval-mode BatchNorm2d, eps 1e-5)
 *   compress_w [128,128] compress_b [128]; gf_w [128,1,K,128] gf_b [128] (from [128,1]);
 *   action_w [5,128] action_b [5] */
typedef struct gpp_planner_weights {
    const float* conv_w[5];
    const float* conv_b[5];
    const float* bn_w[5];
    const float* bn_b[5];
    const float* bn_mean[5];
    const float* bn_var[5];
    const float* compress_w;
    const float* compress_b;
    const float* gf_w;
    const float* gf_b;
    const float* action_w;
    const float* action_b;
} gpp_planner_weights;

/* K = number of graph-filter taps (config.nGraphFilterTaps, decentralplanner.py:131). */
int gpp_planner_create(gpp_planner** out, int K);
void gpp_planner_destroy(gpp_planner* p);

/* Copies/re-lays-out the parameters into the planner's private device arena
 * (k-major conv/linear weights, BatchNorm folded to per-channel scale/shift).
 * `on_device` != 0: the pointers are device pointers, work is enqueued on `stream`;
 * == 0: host pointers (synchronous). Call again whenever the parameters change. */
int gpp_planner_set_weights(gpp_planner* p, const gpp_planner_weights* w, int on_device,
                            void* stream);

/* Device-resident forward.
 *   x       dev f32 [B,N,3,11,11]
 *   S       dev [B,N,N] f32 / f64 (s_is_f64)
 *   logits  dev f32 out [N,B,5]  -- agent-major, so that the reference's Python list of N
 *           tensors [B,5] (decentralplanner.py:303-318) is N contiguous views
 *   features_out  optional dev f32 [B,N,128] node-major CNN+compress features (may be NULL)
 */
int gpp_planner_forward(gpp_planner* p, const float* x, const void* S, int s_is_f64,
                        float* logits, float* features_out, int B, int N, void* stream);

/* Host-buffer forward: H2D copies of x and S, the forward, and the D2H copy of the logits
 * all run on the planner's own stream; returns after the logits are in `logits_host`.
 * This is the call a rollout loop makes once per step (agents/decentralplannerlocal.py
 * :563-580 does the same with .to(device) + model(...)). */
int gpp_planner_forward_host(gpp_planner* p, const float* x_host, const void* S_host,
                             int s_is_f64, float* logits_host, int B, int N);

/* ------------------------------------------------------------------------------------
 * Whole-planner TRAINING forward / backward (replaces DecentralPlannerNet.forward in train mode,
 * decentralplanner.py:278-318, and the autograd pass behind loss.backward(),
 * agents/decentralplannerlocal.py:297-314).  All pointers are device pointers.
 *
 * BatchNorm follows the reference's per-agent semantics: the reference calls ConvLayers once per agent, so
 * batch statistics are over (B,H,W) of one agent's slice and the running statistics receive N sequential
 * momentum updates per forward, in agent order (bn == NULL or NULL members: no running-stat update).
 *   logits   out [N,B,5]                         dlogits  in [N,B,5]  (gradient of the loss)
 *   workspace: gpp_planner_train_workspace_bytes(B,N,K) bytes; written by the forward (saved activations),
 *              read and scribbled on by the backward of the SAME step.
 *   grads: every member is overwritten (not accumulated) with the gradient of the matching parameter.
 * ---------------------------------------------------------------------------------- */
typedef struct gpp_planner_bn_state {
    float* running_mean[5];
    float* running_var[5];
} gpp_planner_bn_state;

typedef struct gpp_planner_grads {
    float* conv_w[5];
    float* conv_b[5];
    float* bn_w[5];
    float* bn_b[5];
    float* compress_w;
    float* compress_b;
    float* gf_w;      /* [128,1,K,128] */
    float* gf_b;      /* [128] */
    float* action_w;
    float* action_b;
} gpp_planner_grads;

size_t gpp_planner_train_workspace_bytes(int B, int N, int K);
int gpp_planner_train_forward(const gpp_planner_weights* w, const gpp_planner_bn_state* bn, float momentum,
                              const float* x, const void* S, int s_is_f64, float* logits, void* workspace,
                              int B, int N, int K, void* stream);
int gpp_planner_train_backward(const gpp_planner_weights* w, const float* x, const void* S, int s_is_f64,
                               const float* dlogits, void* workspace, const gpp_planner_grads* g,
                               int B, int N, int K, void* stream);

/* Fused training loss (replaces the per-agent loop of agents/decentralplannerlocal.py:305-312 and its autograd graph):
 *   loss = (1/N) sum_i CrossEntropy(logits[i], argmax_a target[:, i, a])          (mean over the batch per agent)
 *   dlogits[i,b,:] = grad_scale * (softmax(logits[i,b,:]) - onehot) / (N*B)       (NULL to skip)
 *   logits dev f32 [N,B,5] (as gpp_planner_forward / _train_forward write them); target_onehot dev [B,N,5], int64
 *   (target_is_i64 != 0, the dataloader's format) or f32; loss dev f32 [1].  One launch, deterministic. */
int gpp_planner_ce_loss(const float* logits, const void* target_onehot, int target_is_i64, float* loss,
                        float* dlogits, float grad_scale, int B, int N, void* stream);

/* ------------------------------------------------------------------------------------
 * GPU-resident rollout step, B episodes in lock-step (what surrounds the forward in the reference's
 * rollout loop, agents/decentralplannerlocal.py:560-592; the reference runs it on the host, one episode
 * at a time).  All pointers are device pointers; positions are integer cells (x, y) and never leave the
 * device between steps.
 *
 * gpp_rollout_build_inputs replaces multiRobotSim.getCurrentState (utils/multirobotsim_dcenlocal.py:425-453
 * -> AgentState.toInputTensor, dataloader/statetransformer.py:82-130) and multiRobotSim.getGSO (:367-394 ->
 * computeAdjacencyMatrix :320-365, connectivity test graphTools.py:396-423):
 *   pos, goal  [B,N,2] int32      map [B,W,W] or (map_shared) [W,W] uint8, 1 = obstacle
 *   radius     [B] f64 in/out: communication radius.  grow_radius != 0 (the reference's step 0): radius is divided by
 *              1.1 once, then multiplied by 1.1 until the graph is connected, and written back.
 *   x          out f32 [B,N,3,11,11]   S out [B,N,N] f64 (s_is_f64, as the simulator emits) or f32
 *   connected  out [B] int32 or NULL
 * Bit-exact with the reference (integer window arithmetic; the GSO is IEEE float64 sqrt / divide / multiply).
 *
 * gpp_rollout_move replaces multiRobotSim.move (:562-723) incl. interRobotCollision (:462-555):
 *   logits [N,B,5] (as the planner writes them); action = first maximum (LogSoftmax + argmax, :589-591); moves into
 *   the map edge or an obstacle become "stay"; vertex conflicts and position swaps are resolved as the reference does.
 *   Where the reference draws random.choice(collided agents), the contract here is round-robin: the c-th draw of the
 *   episode picks collided[c % len] (agent order); c is choice_counter[b].
 *   pos in/out; reached / start_step / end_step [B,N] in/out (-1 = not yet); last_action [B,N] out; maxstep [B];
 *   active [B] or NULL (0 = leave the episode untouched); flags [B,3] out = {all agents had reached their goal before
 *   this move, check_moveCollision, check_predictCollsion}; currentstep = 1-based step index (:561). */
int gpp_rollout_build_inputs(const int* pos, const int* goal, const unsigned char* map, int map_shared,
                             double* radius, int grow_radius, float* x, void* S, int s_is_f64,
                             int* connected, int B, int N, int W, void* stream);
int gpp_rollout_move(const float* logits, int* pos, const int* goal, const unsigned char* map, int map_shared,
                     const int* maxstep, const int* active, int* reached, int* start_step, int* end_step,
                     int* last_action, unsigned int* choice_counter, int* flags, int currentstep, int B, int N,
                     int W, void* stream);

/* ------------------------------------------------------------------------------------
 * Batched evaluation: the scoring half of agents/decentralplannerlocal.py:535-648 (mutliAgent_ActionPolicy) for B
 * episodes advanced with gpp_rollout_move.  All pointers are device pointers, int32.
 *
 * gpp_rollout_expert_metrics replaces multiRobotSim.getPathTarget (utils/multirobotsim_dcenlocal.py:159-230); run once.
 *   start, goal [B,N,2]; expert_action [B,N,T] action indices (0 up, 1 left, 2 down, 3 right, 4 stop).
 *   Each agent replays its T actions from its start, ignoring obstacles and other agents.  startStep = first step
 *   whose action is not stop; endStep = step + 1 at the first arrival on the goal.
 *   makespan_target [B] = max(endStep) - min(startStep), flowtime_target [B] = sum(endStep - startStep), target_valid [B]
 *   = 1 when both are usable as divisors: every agent arrives, every agent moves (the reference computes end - None
 *   otherwise), all actions are in 0..4 and neither target is 0.  Unusable targets are written as 0, which is also
 *   what the reference keeps when some agent never arrives.
 *
 * gpp_rollout_record: the per-step bookkeeping of mutliAgent_ActionPolicy (:555-624); call it after every
 * gpp_rollout_move with the same active, flags and currentstep.  Episodes with active[b] == 0 are skipped (their flags
 * are stale).  For the others the collision flags are OR-ed into the record; the episode ends when flags[b][0] (all
 * agents had reached their goals before the move) is set or currentstep >= maxstep[b].  Then the whole row of
 * outcome[b] is written and active[b] is cleared.
 *   outcome [B, GPP_OUTCOME_FIELDS]: zero it before the first step.
 *   makespan_target / flowtime_target: [B] from gpp_rollout_expert_metrics, or makespan_target == NULL when no expert
 *   is given (the target columns and GPP_OUTCOME_FIND_OPTIMAL are then 0).
 * The columns follow the reference, quirks included:
 *   MAKESPAN_PREDICT / FLOWTIME_PREDICT = max(end) - min(start) / sum(end - start) of the last move only when
 *     checkOptimality ran (collision-free success, or currentstep >= maxstep); otherwise the pre-loop defaults
 *     maxstep / maxstep * N of getOptimalityMetrics (:555).
 *   FIND_OPTIMAL = collision-free success with predicted <= target on both, reset to 0 when currentstep >= maxstep.
 *   ALL_REACH_GOAL is flags[b][0] of the last move: agents that arrive on the maxstep move do not count.
 *   NO_REACH_GOAL_SH = timeout and not ALL_REACH_GOAL and COLLISION_PREDICTED and not COLLISION_HAPPENED.
 *   COLLISION_FREE = ALL_REACH_GOAL and not COLLISION_HAPPENED.   STEPS = the final currentStep.
 *   VALID = 1 once the episode has ended and the reference would score it without raising: every predicted start step
 *     is defined and (with targets) both targets are nonzero.
 * ---------------------------------------------------------------------------------- */
typedef enum gpp_outcome_field {
    GPP_OUTCOME_STEPS = 0,
    GPP_OUTCOME_ALL_REACH_GOAL = 1,
    GPP_OUTCOME_NO_REACH_GOAL_SH = 2,
    GPP_OUTCOME_FIND_OPTIMAL = 3,
    GPP_OUTCOME_COLLISION_FREE = 4,
    GPP_OUTCOME_COLLISION_PREDICTED = 5,
    GPP_OUTCOME_COLLISION_HAPPENED = 6,
    GPP_OUTCOME_NUM_REACH_GOAL = 7,
    GPP_OUTCOME_MAKESPAN_PREDICT = 8,
    GPP_OUTCOME_MAKESPAN_TARGET = 9,
    GPP_OUTCOME_FLOWTIME_PREDICT = 10,
    GPP_OUTCOME_FLOWTIME_TARGET = 11,
    GPP_OUTCOME_VALID = 12,
    GPP_OUTCOME_FIELDS = 13
} gpp_outcome_field;

/* replaces multiRobotSim.getPathTarget (utils/multirobotsim_dcenlocal.py:159-230) */
int gpp_rollout_expert_metrics(const int* start, const int* goal, const int* expert_action, int T,
                               int* makespan_target, int* flowtime_target, int* target_valid, int B, int N, void* stream);
/* per-step outcome bookkeeping of mutliAgent_ActionPolicy (agents/decentralplannerlocal.py:555-624) */
int gpp_rollout_record(const int* flags, const int* maxstep, const int* reached, const int* start_step,
                       const int* end_step, const int* makespan_target, const int* flowtime_target,
                       int* active, int* outcome, int currentstep, int B, int N, void* stream);

/* ------------------------------------------------------------------------------------
 * Device-resident expert dataset: the training samples the reference's online-expert DataTransformer writes as one
 * .mat file per case (onlineExpert/DataTransformer_local_onlineExpert.py:154-305) and its loader slices into one sample
 * per step (dataloader/Dataloader_dcplocal_notTF_onlineExpert.py:142-157), built on demand from integer states.
 * All pointers are device pointers.  The cases share N (2 <= N <= 64, else GPP_ERR_UNSUPPORTED) and the map size W.
 *   states       [R,N,2] int32: the T = makespan + 1 states of every case, case after case (agent i at step t is at
 *                its path's cell t while t < len(path), at its goal after that)
 *   case_offset  [C] int32: row of each case's step 0;  case_steps [C] int32: its T
 *   goal         [C,N,2] int32
 *
 * gpp_expert_radius replaces computeAdjacencyMatrix (:256-305) and the move check of obtainSchedule (:177-189); run
 * once per case.  radius [C] f64 out: init_radius (the transformer's constant 5) multiplied by 1.1 at every step, in
 * order, that is not connected under the current value (the value carries over to the next step).  valid [C] int32
 * out: 1 when every move state[t] -> state[t+1] (the goal after the last state) is one of the five deltas; bad [C,2]
 * int32 out: (step, agent) of the first other move in the reference's order (agent after agent), else (-1, -1).
 *
 * gpp_expert_gather: B samples, sample = state row (step t of case c is row case_offset[c] + t).
 *   row_case [R] int32: case of every row;  map [C,W,W] uint8, 1 = obstacle;  radius [C] from gpp_expert_radius
 *   rows [B] int64: the samples; a row outside 0..R-1 leaves its outputs unwritten
 *   x             out f32 [B,N,3,11,11] or NULL: AgentState.toSeqInputTensor at the sample's state
 *   target_onehot out int64 [B,N,5] or NULL: the one-hot action state[t] -> state[t+1] (the goal after the last state)
 *   S             out [B,N,N] f64 (s_is_f64) or f32, or NULL: D^-1/2 A D^-1/2, A = (pdist < radius[c]) with a zero
 *                 diagonal, computed in float64 (f32 = rounded, as the loader's .float())
 * Bit-exact with the reference for the cases gpp_expert_radius marks valid.
 * ---------------------------------------------------------------------------------- */
int gpp_expert_radius(const int* states, const int* case_offset, const int* case_steps, const int* goal,
                      double init_radius, double* radius, int* valid, int* bad, int C, int N, void* stream);
int gpp_expert_gather(const int* states, const int* case_offset, const int* case_steps, const int* row_case,
                      const int* goal, const unsigned char* map, const double* radius, const long long* rows,
                      float* x, long long* target_onehot, void* S, int s_is_f64, int B, int N, int W, int R,
                      void* stream);

/* ------------------------------------------------------------------------------------
 * Batched expert solver (replaces the reference's prebuilt `ecbs -w 1.1` binary, run by onlineExpert/ECBS_onlineExpert.py
 * on the online expert's failure cases and by offlineExpert/CasesGenerator.py:283-340 on the offline dataset).
 * Conflict-based search (CBS) minimising the sum of costs (SoC): the SoC it returns is optimal among the solutions with
 * makespan <= H, which meets ECBS's guarantee (SoC <= w x optimal).  One warp per case, C cases per call.
 *
 * Move model (the reference simulator's): the five actions up (-1,0), left (0,-1), down (1,0), right (0,1), stop;
 * obstacles and the map edge are blocked; two agents on one cell at one step (vertex conflict) and two agents trading
 * cells in one step (swap conflict) are forbidden; an agent stays on its goal after its path ends.  Agent i's cost tau_i
 * is the step after which it stays on its goal; the case's makespan is max tau_i.
 *
 * Every tie is fixed, so the solution is a function of the input:
 *   low level (agent i under its constraints): L_0 = {start}; L_{t+1} = the free cells v not vertex-constrained at t+1
 *     with some u in L_t, v in {u, u + delta}, (u -> v, t) not edge-constrained.  tau_i = the smallest t <= H with
 *     goal in L_t and t > the latest vertex constraint on the goal (or -1); none: the node is infeasible.  The path is
 *     backtracked from (goal, tau_i): at each step the first predecessor p in L_{t-1} whose move p -> c is not
 *     edge-constrained, trying the actions in the order stop, up, left, down, right (p = c - delta).
 *   conflict: the earliest t; at that t vertex conflicts (pairs i < j, lexicographic) before swap conflicts between t
 *     and t+1 (i < j, lexicographic); paths are extended with their goal.
 *   high level: expand the open node with the smallest (SoC, creation index); the root has index 0.  The child that
 *     constrains i is created before the one that constrains j: a vertex conflict at (v, t) adds the vertex constraint
 *     (v, t); a swap with i moving u -> v adds (u -> v, t) for i and (v -> u, t) for j.  Only the constrained agent is
 *     replanned; an infeasible child is not created and takes no index.
 *   stop: GPP_SOLVE_SOLVED when the expanded node has no conflict; GPP_SOLVE_NO_SOLUTION when an agent of the root is
 *     infeasible or the open list runs empty (no solution has makespan <= H); GPP_SOLVE_BUDGET when a feasible child
 *     would be node number max_nodes + 1.
 *
 * All pointers are device pointers.  Envelope: 1 <= N <= 64, 1 <= W <= 64, 1 <= H <= 1024, 1 <= max_nodes <= 65536,
 * else GPP_ERR_UNSUPPORTED.  The caller guarantees distinct starts, distinct goals and free in-map cells.
 *   map [C,W,W] uint8 (nonzero = obstacle);  start, goal [C,N,2] int32 cells (x, y)
 *   status [C] (gpp_solve_status);  soc, makespan [C] (-1 unless solved)
 *   nodes_created, nodes_expanded [C] (the root counts as created, the solved node as expanded)
 *   low_level [C]: single-agent searches run (the root's, stopping at the first infeasible agent, and one per child)
 *   tau [C,N] (-1 unless solved);  paths [C,N,H+1] int16: agent i's cell x * W + y at every step, the goal after
 *   tau_i (-1 unless solved)
 *   workspace: gpp_expert_solve_workspace_bytes(C, N, W, H, max_nodes) bytes of device scratch.  It is sized per
 *   resident warp, not per case: 256 + warps * per-warp bytes, warps = min(C, resident warps, 2 GiB / per-warp bytes),
 *   per-warp bytes = 8 W (H+1) layers + 56 max_nodes (nodes, open list, constraints) + 2 (N + max_nodes)(H+1) paths,
 *   each part rounded up to 256 bytes.
 * ---------------------------------------------------------------------------------- */
typedef enum gpp_solve_status {
    GPP_SOLVE_SOLVED = 0,
    GPP_SOLVE_NO_SOLUTION = 1,
    GPP_SOLVE_BUDGET = 2
} gpp_solve_status;

/* 0 outside the envelope or for C <= 0 */
size_t gpp_expert_solve_workspace_bytes(int C, int N, int W, int H, int max_nodes);
int gpp_expert_solve(const unsigned char* map, const int* start, const int* goal, int H, int max_nodes,
                     int* status, int* soc, int* makespan, int* nodes_created, int* nodes_expanded, int* low_level,
                     int* tau, short* paths, void* workspace, size_t workspace_bytes, int C, int N, int W,
                     void* stream);

/* ------------------------------------------------------------------------------------
 * Expert case generation (replaces offlineExpert/CasesGenerator.py's mapGen, img_fill and setup_cases): K candidates
 * per call, numbered first_candidate, first_candidate + 1, ...  A candidate is a W x W maze, its filled map and N
 * (start, goal) pairs.  Its randomness is a pure function of (seed, k), so the result does not depend on the launch.
 *
 * Draws: Philox4x32-10, key (seed & 0xffffffff, seed >> 32), counter (k & 0xffffffff, k >> 32, block, phase); phase 0
 *   is the maze, phase 1 the agents.  Draw j of a phase is word j % 4 of block j / 4.  A bounded draw in [0, n) is
 *   (u32 * n) >> 32 in 64-bit arithmetic, no rejection.
 * Maze (mapGen with height = width = W): all free; aisles times: col = 2 draw(W/2), then row = 2 draw(W/2), mark
 *   (row, col); then walk steps, each building the neighbour list (row, col-2) if col > 1, (row, col+2) if col < W-2,
 *   (row-2, col) if row > 1, (row+2, col) if row < W-2.  A non-empty list picks list[draw(len - 1)] (the last entry is
 *   never picked); a free pick is marked with the cell between and becomes the position.  An empty list draws nothing.
 *   aisles = int(density * ((W//2) * (W//2))) and walk = int(complexity * (5 * (W + W))) are the caller's.
 * Fill (img_fill): the free cells are the 4-connected free component of the maze containing (0, 0); every other cell
 *   is an obstacle.  If (0, 0) is an obstacle there are no free cells.
 * Agents (random.sample(free cells, 2) per agent): F free cells in row-major order; agent i draws s = draw(F) (phase-1
 *   word 2i) and g' = draw(F - 1) (word 2i + 1); goal index g = g' + (g' >= s).  Cells are (x, y) = (row, col).
 * Status: GPP_CASE_TOO_FEW_FREE when F < 2, GPP_CASE_SHARED_CELL when two agents share a start or a goal,
 *   GPP_CASE_ACCEPTED otherwise.
 *
 * All pointers are device pointers.  Envelope: 1 <= N <= 64, 2 <= W <= 64, aisles * (2 + walk) < 2^31, else
 * GPP_ERR_UNSUPPORTED.
 *   map [K,W,W] uint8 out: the filled map, 1 = obstacle
 *   start, goal [K,N,2] int32 out: cells (x, y); -1 for a GPP_CASE_TOO_FEW_FREE candidate
 *   status [K] int32 out (gpp_case_status)
 * ---------------------------------------------------------------------------------- */
typedef enum gpp_case_status {
    GPP_CASE_ACCEPTED = 0,
    GPP_CASE_TOO_FEW_FREE = 1,
    GPP_CASE_SHARED_CELL = 2
} gpp_case_status;

int gpp_case_generate(unsigned long long seed, unsigned long long first_candidate, int K, int N, int W, int aisles,
                      int walk, unsigned char* map, int* start, int* goal, int* status, void* stream);

/* Asynchronous variant for pipelined rollouts over INDEPENDENT episode batches: stages the inputs on a copy stream,
 * enqueues the forward on one of the planner's four compute streams (tickets rotate over them, so the feature kernel of
 * one batch runs next to the kernels of the batches before it on the SMs they leave idle) and returns at once with a completion ticket; the
 * host buffers MUST be pinned and must stay untouched until gpp_planner_wait(ticket) returns.  Consecutive tickets may
 * complete in either order -- wait for the ticket whose logits are needed; at most 16 tickets may be outstanding. */
int gpp_planner_forward_host_async(gpp_planner* p, const float* x_host, const void* S_host,
                                   int s_is_f64, float* logits_host, int B, int N,
                                   unsigned long long* ticket);
int gpp_planner_wait(gpp_planner* p, unsigned long long ticket);

/* The same pipelining for DEVICE tensors (a driver advancing several independent episode batches whose inputs are produced on
 * the GPU): x / S must be complete in `stream` order at the time of the call (an event is recorded there), the forward
 * runs on the next compute lane, and the logits (device memory, [N][B][5]) may be consumed after
 * gpp_planner_join(p, ticket, consumer_stream) -- a device-side wait, the host does not block -- or after
 * gpp_planner_wait(ticket).  x, S and logits must stay untouched until then; tickets share the numbering and the limit of
 * 16 outstanding calls with gpp_planner_forward_host_async.  Replaces a loop of `model.addGSO(S); model(x)` calls
 * (gnn_pathplanning/agents/decentralplannerlocal.py:576-588) over independent batches. */
int gpp_planner_forward_async(gpp_planner* p, const float* x, const void* S, int s_is_f64, float* logits, int B, int N,
                              void* stream, unsigned long long* ticket);
int gpp_planner_join(gpp_planner* p, unsigned long long ticket, void* stream);

/* Which graph-filter kernel the planner uses: 0 = automatic (tensor cores once B*N >= 4096 node
 * rows), 1 = CUDA-core fp32 kernel (gf_fwd_kernel), 2 = wgmma 3xTF32 kernel (gf_fwd_tc_kernel),
 * 3 = wgmma pair fp16-split kernel (gf_fwd_pair_kernel).  GPP_ERR_UNSUPPORTED at forward
 * time if N / K are outside the requested kernel's envelope. */
int gpp_planner_set_graph_filter_mode(gpp_planner* p, int mode);

/* Which feature-extractor (CNN + compress MLP) kernel the planner uses: 0 = automatic (currently always the
 * CUDA-core kernel, the faster one at every measured size), 1 = CUDA-core fp32 kernel (feature_kernel),
 * 2 = wgmma 3xTF32 implicit-GEMM kernel (feature_tc_kernel). */
int gpp_planner_set_feature_mode(gpp_planner* p, int mode);

/* Per-kernel device timing for the roofline report: when enabled, gpp_planner_forward records
 * CUDA events before / between / after its two kernels on the launching stream (at most 8192
 * steps are kept).  gpp_planner_get_profile synchronises on the recorded events, returns the
 * summed durations in milliseconds and the number of steps they cover, and clears the log. */
int gpp_planner_set_profiling(gpp_planner* p, int enable);
int gpp_planner_get_profile(gpp_planner* p, double* feature_ms, double* graph_filter_ms, int* steps);

/* Number of kernels of this library launched by this process (any thread) since
 * the last reset (bench.py's gpu_launches claim is read from here, not guessed). */
unsigned long long gpp_launch_count(void);
void gpp_reset_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* GNNPP_B200_H */
