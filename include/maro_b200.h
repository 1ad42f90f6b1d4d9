/*
 * maro_b200.h — C ABI of the H100-native batched discrete-event simulation core.
 *
 * This is the drop-in boundary (SURVEY.md §8b, seam 3): everything `maro.simulator.Env` /
 * `maro.vector_env.VectorEnv` need from the step path, for B independent replicas at once, as plain
 * pointers and sizes.  No torch / Python types.  The reference has no C ABI for this path (its seams are a
 * Cython vtable and Python classes); each entry point cites the reference interface it replaces.
 *
 * Conventions
 *   - Every function returns 0 on success, non-zero on failure; maro_last_error() returns the message of
 *     the last failure on the calling thread.
 *   - The caller owns every in/out buffer; the library owns device memory, streams and snapshot rings.
 *     No pointer handed out by the library outlives maro_cim_destroy().
 *   - A handle is NOT thread-safe (the reference Env is single-threaded: maro/simulator/core.py:20).
 *   - "host" entry points take host buffers and perform H2D / D2H inside the call; "_device" entry points
 *     take device pointers and only enqueue work on the handle's stream.
 */
#ifndef MARO_B200_H
#define MARO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MARO_B200_ABI_VERSION 2

/* ------------------------------------------------------------------------------------------------
 * Static tables of one CIM topology instance (config + max_tick + seed).
 * Produced on the host by maro_b200.scenarios.cim.topology.build_topology(), which restates
 * maro/data_lib/cim/cim_data_generator.py:18-205 and maro/data_lib/cim/parsers.py:14-211.
 * All arrays are caller-owned and copied during maro_cim_create().
 * ---------------------------------------------------------------------------------------------- */
typedef struct MaroCimTopology {
    int32_t n_ports, n_vessels, n_routes;
    int32_t past_stop_number, future_stop_number; /* config "stop_number"                            */
    int32_t max_tick;                             /* start_tick + durations                          */
    int32_t order_mode;                           /* 0 = fixed, 1 = unfixed (entities.py:74-84)      */
    int32_t total_containers;
    double container_volume;                      /* config container_volumes[0]                     */
    /* ports [n_ports] */
    const int32_t* port_capacity;
    const int32_t* port_init_empty;
    const double* full_return_base;
    const double* full_return_noise;
    const double* empty_return_base;
    const double* empty_return_noise;
    const double* source_base;
    const double* source_noise;
    const int32_t* target_offset; /* [n_ports + 1] into target_* */
    const int32_t* target_port;
    const double* target_base;
    const double* target_noise;
    /* vessels [n_vessels] */
    const int32_t* vessel_capacity;
    const int32_t* vessel_init_empty;
    const int32_t* vessel_route;
    const int32_t* vessel_period;      /* vessel_period_without_noise (cim_data_container.py:218-229)    */
    const int32_t* vessel_route_start; /* index of the start port inside the vessel's route             */
    const int32_t* vessel_leg_offset;  /* [n_vessels + 1] into vessel_leg                                */
    const int32_t* vessel_leg;         /* parking duration + ceil(distance / speed) per route position  */
    const int32_t* stop_offset;        /* [n_vessels + 1] into stop_*                                    */
    const int32_t* stop_arrival;
    const int32_t* stop_leave;
    const int32_t* stop_port;
    /* routes */
    const int32_t* route_offset; /* [n_routes + 1] into route_port */
    const int32_t* route_port;
    /* per-tick order budget, [max_tick] (parsers.py:63-107) */
    const int32_t* order_proportion;
    /* MT19937 seeds of the two in-step random streams (sim_random.py:48-63). */
    uint32_t order_number_seed;
    uint32_t buffer_time_seed;
} MaroCimTopology;

typedef struct MaroCimConfig {
    int32_t n_replicas;
    int32_t start_tick;          /* Env(start_tick=)            core.py:46                            */
    int32_t snapshot_resolution; /* Env(snapshot_resolution=)   core.py:48                            */
    int32_t max_snapshots;       /* Env(max_snapshots=), <=0: keep every frame  core.py:49            */
    int32_t device;              /* CUDA device ordinal                                               */
    int32_t queue_capacity;      /* per-replica dynamic-event slots; <=0: library default             */
    int32_t max_actions;         /* actions per replica per step (A_MAX); <=0: 1                      */
    const int32_t* replica_topology; /* [n_replicas] index into topos[], NULL: all 0                  */
    int32_t decision_mode;       /* 0 Sequential, 1 Joint (Env(decision_mode=), core.py:354-366; CIM only): a step returns EVERY
                                    decision event of the tick — n_vessels rows of MARO_CIM_DECISION_WORDS per replica, the list
                                    ends before the first row whose status is not MARO_STATUS_DECISION — and takes one action row
                                    per decision in the same order (type MARO_ACTION_NONE = None; fewer rows = the rest unanswered) */
} MaroCimConfig;
enum { MARO_ACTION_NONE = 2 }; /* third value of the action row's type word (MARO_ACTION_LOAD / _DISCHARGE below) */

/* Row layout of the decision output, one row of MARO_CIM_DECISION_WORDS int32 per replica.
 * Mirrors DecisionEvent (maro/simulator/scenarios/cim/common.py:72-150) + step status. */
enum {
    MARO_DEC_TICK = 0,
    MARO_DEC_PORT = 1,
    MARO_DEC_VESSEL = 2,
    MARO_DEC_SCOPE_LOAD = 3,      /* ActionScope.load      = min(port.empty, vessel.remaining_space) */
    MARO_DEC_SCOPE_DISCHARGE = 4, /* ActionScope.discharge = vessel.empty                            */
    MARO_DEC_EARLY_DISCHARGE = 5,
    MARO_DEC_STATUS = 6,          /* MARO_STATUS_*                                                   */
    MARO_DEC_STEP = 7,            /* ordinal of this env-step inside the episode (0 = first decision)  */
    MARO_CIM_DECISION_WORDS = 8
};

enum {
    MARO_STATUS_DECISION = 0, /* (metrics, decision, False)                     core.py:350            */
    MARO_STATUS_DONE = 1,     /* (metrics, None, True) — episode just ended     core.py:381            */
    MARO_STATUS_FINISHED = 2, /* (None, None, True) — stepping a finished env   core.py:128-131        */
    MARO_STATUS_INACTIVE = 3, /* replica not selected by the active mask (VectorEnv dict stepping)     */
    MARO_STATUS_BAD_ACTION = -1,   /* the reference would raise AssertionError (business_engine.py:731,736) */
    MARO_STATUS_QUEUE_OVERFLOW = -2
};

/* Action row: 4 int32 {vessel_idx, port_idx, quantity, action_type}; Action in cim/common.py:25-53. */
enum { MARO_ACTION_LOAD = 0, MARO_ACTION_DISCHARGE = 1, MARO_CIM_ACTION_WORDS = 4 };

/* Metrics row: 3 int64 {order_requirements, container_shortage, operation_number};
 * CimBusinessEngine.get_metrics, business_engine.py:270-282. */
enum { MARO_CIM_METRIC_WORDS = 3 };

/* Node types for snapshot queries (frame_builder.py:11-33). */
enum { MARO_CIM_NODE_PORTS = 0, MARO_CIM_NODE_VESSELS = 1, MARO_CIM_NODE_MATRICES = 2 };

typedef struct MaroCimEnv MaroCimEnv;

const char* maro_last_error(void);
int maro_abi_version(void);

/* Env.__init__ / VectorEnv.__init__ (core.py:42-90, vector_env.py:55-93): allocate B replicas on one GPU. */
int maro_cim_create(const MaroCimTopology* topos, int32_t n_topos, const MaroCimConfig* cfg, MaroCimEnv** out);
/* VectorEnv.stop / __del__ (vector_env.py:146-160). */
int maro_cim_destroy(MaroCimEnv* env);
/* Stream for all subsequent work.  external != 0: use `cuda_stream` (a cudaStream_t; 0 is the legacy default
 * stream, e.g. torch's default current stream).  external == 0: back to the library's own stream. */
int maro_cim_set_stream(MaroCimEnv* env, void* cuda_stream, int32_t external);

/* Env.step / VectorEnv.step (core.py:92-133, vector_env.py:116-144), host buffers.
 *   active      [B] uint8 or NULL (all)            — dict/subset stepping of VectorEnv
 *   actions     [B][max_actions][4] int32 or NULL  — NULL = step(None) for every replica
 *   n_actions   [B] int32 or NULL (NULL with actions != NULL means 1 each)
 *   decisions   [B][8] int32 out, metrics [B][3] int64 out                                           */
int maro_cim_step(MaroCimEnv* env, const uint8_t* active, const int32_t* actions, const int32_t* n_actions,
                  int32_t* decisions, int64_t* metrics);
/* Zero host-copy variant: the library's own pinned (and device-mapped) staging buffers, laid out exactly like the
 * arguments of maro_cim_step.  Fill actions / n_actions / active in place, call maro_cim_step_pinned with flags saying
 * which inputs are present, read decisions / metrics in place.  The pointers stay valid until maro_cim_destroy. */
int maro_cim_pinned_buffers(MaroCimEnv* env, void** actions, void** n_actions, void** active, void** decisions,
                            void** metrics);
int maro_cim_step_pinned(MaroCimEnv* env, int32_t use_actions, int32_t use_n_actions, int32_t use_active);
/* Resident mode, host agents: when every replica block of the handle fits on the chip at once, maro_cim_step and
 * maro_cim_step_pinned drive a kernel that STAYS resident between calls (replica blocks in shared memory): per call the
 * host writes one 16-byte command row per replica into mapped pinned memory, the replica's warp picks it up, steps and
 * writes its decision / metrics rows back; no launch, no stage-in / write-back, no stream synchronisation per step.  The
 * kernel leaves on its own once the host has been outside submit / wait for about two MARO_B200_IDLE_US periods (default
 * 200 us each; the host side bumps a heartbeat word while it is inside them) and whenever another entry point needs the
 * state in device memory.  MARO_B200_SESSION=0 disables it (one launch per call, as for large
 * batches).
 * Asynchronous halves of maro_cim_step_pinned for a contiguous replica range (what VectorEnv's dict stepping gives the
 * reference, vector_env.py:131-144, without blocking): submit sends the step to replicas [first, first + count) and returns
 * at once, wait blocks until their decision / metrics rows are in the pinned buffers.  Ranges are whole blocks of
 * maro_cim_pinned_granularity() replicas (0: the batch is not resident, only maro_cim_step_pinned is available); a host
 * agent overlaps its own work on one range with the device's work on the others.
 * Threads: submit / wait / maro_cim_reset(mask) may be called concurrently from several host threads as long as the replica
 * ranges (mask bits) of the threads are disjoint; every other entry point of a handle is single-threaded. */
int32_t maro_cim_pinned_granularity(MaroCimEnv* env);
int maro_cim_submit_pinned(MaroCimEnv* env, int32_t first, int32_t count, int32_t use_actions, int32_t use_n_actions,
                           int32_t use_active);
int maro_cim_wait_pinned(MaroCimEnv* env, int32_t first, int32_t count);
/* Same, device pointers, asynchronous on the handle's stream (no host<->device copies). */
int maro_cim_step_device(MaroCimEnv* env, const uint8_t* d_active, const int32_t* d_actions,
                         const int32_t* d_n_actions, int32_t* d_decisions, int64_t* d_metrics);

/* Env.reset (core.py:143-170) for the replicas selected by mask (NULL = all).  Tables of the replicas'
 * topologies must already be resident (see maro_cim_set_topology for keep_seed=False / set_seed).  While the resident
 * kernel is live the reset costs nothing here: it rides on each replica's next command row and is carried out in shared
 * memory (any call that reads device state applies what is still pending first).  The mask is read during the call; no
 * pinned staging buffer (maro_cim_pinned_buffers) is written, so inputs filled there for the next step survive a reset. */
int maro_cim_reset(MaroCimEnv* env, const uint8_t* mask);
/* Replace topology slot `index` (same shape) — used for reset(keep_seed=False) and Env.set_seed. */
int maro_cim_set_topology(MaroCimEnv* env, int32_t index, const MaroCimTopology* topo);

/* env.snapshot_list[node][ticks:nodes:attrs] (frame.pyx:754-801, np_backend.pyx:520-549), static-backend
 * semantics: out[replica][tick][node][attr][slot] as float64, frames not in the ring -> zeros.
 * `frame_indices` are snapshot frame indices (tick // resolution), attrs are attribute ids from
 * maro_cim_attr_id().  Returns the number of doubles written per replica through *out_per_replica. */
int maro_cim_query(MaroCimEnv* env, const int32_t* replicas, int32_t n_replicas, int32_t node_type,
                   const int32_t* frame_indices, int32_t n_frames, const int32_t* nodes, int32_t n_nodes,
                   const int32_t* attrs, int32_t n_attrs, double* out, int64_t* out_per_replica);
/* Same gather, output left in device memory (float64). */
int maro_cim_query_device(MaroCimEnv* env, const int32_t* replicas, int32_t n_replicas, int32_t node_type,
                          const int32_t* frame_indices, int32_t n_frames, const int32_t* nodes,
                          int32_t n_nodes, const int32_t* attrs, int32_t n_attrs, double* d_out,
                          int64_t* out_per_replica);
/* Result layout of maro_*_query / maro_cim_query_device for this handle — the reference picks its backend per process
 * (DEFAULT_BACKEND_NAME, maro/backends/frame.pyx:60-66) and the two backends answer queries differently:
 *   MARO_QUERY_LAYOUT_STATIC  (default; NumpyBackend, np_backend.pyx:520-549): [frame][node][attr][slot] packed, frames not in
 *                             the ring read as 0, values exact;
 *   MARO_QUERY_LAYOUT_DYNAMIC (RawBackend, raw/snapshotlist.cpp:244-318, _raw_backend_.pyx:263-315): every attribute padded to
 *                             max_slots = the widest queried attribute, i.e. [frame][node][attr][max_slots]; missing slots and
 *                             frames not in the ring are NaN; values pass through float32 (ATTR_FLOAT).
 * `out_per_replica` of the query calls reports the per-replica element count of the active layout. */
enum { MARO_QUERY_LAYOUT_STATIC = 0, MARO_QUERY_LAYOUT_DYNAMIC = 1 };
/* Device-state checkpoint — what the reference leaves unimplemented in Env.dump ("Dump environment for restore",
 * maro/simulator/core.py:135-141): the complete simulation state of the handle (replica blocks incl. event queues, snapshot
 * ring, RNG streams, topology tables) goes to one file; `load` restores it into a handle created with the same topologies /
 * configuration (checked) and the episode continues bit for bit.  with_snapshots = 0 leaves the ring rows out (the ring then
 * restarts empty after a load). */
int maro_cim_save(MaroCimEnv* env, const char* path, int32_t with_snapshots);
int maro_cim_load(MaroCimEnv* env, const char* path);
int maro_cim_set_query_layout(MaroCimEnv* env, int32_t layout);
/* Attribute id / slot count by name for a node type; -1 if unknown. */
int32_t maro_cim_attr_id(MaroCimEnv* env, int32_t node_type, const char* name);
int32_t maro_cim_attr_slots(MaroCimEnv* env, int32_t node_type, int32_t attr_id);

/* env.current_frame (core.py:190-193): copy the live frame words of one replica to the host. */
int maro_cim_read_frame(MaroCimEnv* env, int32_t replica, int32_t* out_words, int32_t n_words);
int32_t maro_cim_frame_words(MaroCimEnv* env);
/* env.tick (core.py:196-198) for all replicas. */
int maro_cim_ticks(MaroCimEnv* env, int32_t* out_ticks);
/* Cumulative per-replica work counters {env_steps, ticks, events, snapshots} as int64[B][4]. */
int maro_cim_counters(MaroCimEnv* env, int64_t* out);
/* Frame indices currently held by the snapshot ring of one replica (SnapshotList.get_frame_index_list). */
int maro_cim_snapshot_frames(MaroCimEnv* env, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out);

/* Agent helper used by bench.py: the hello-world random policy (examples/hello_world/cim/hello.py:24-32)
 * as a counter-based hash of (replica_base + replica, decision ordinal = decisions[r][MARO_DEC_STEP]), evaluated
 * on the device so the env state never leaves HBM (and the step loop can be captured in a CUDA graph). */
int maro_cim_random_policy_device(MaroCimEnv* env, const int32_t* d_decisions, int32_t* d_actions,
                                  uint32_t seed, uint32_t replica_base);

/* Resident mode, device agents: `n_steps` fused Env.step calls per replica in ONE launch.  The replica block is staged
 * into shared memory once, the agent is a device callback evaluated between the steps (policy 0 = step(None) every
 * time, 1 = the hashed hello-world agent of maro_cim_random_policy_device with the same seed / replica_base), the block
 * is written back once.  Equivalent, row for row, to n_steps x {policy kernel; maro_cim_step_device}:
 *   d_decisions [B][8] in/out — in: the rows the previous call returned (they feed the agent), out: the last rows
 *   d_metrics   [B][3] out
 *   d_trace     [n_steps][B][8] out or NULL — the decision row of every fused step (replicas that finish early repeat
 *               their MARO_STATUS_FINISHED row)
 * Replaces the loop of examples/hello_world/cim/hello.py:21-35 around Env.step (core.py:92-133). */
int maro_cim_rollout_device(MaroCimEnv* env, int32_t policy, uint32_t seed, uint32_t replica_base, int32_t n_steps,
                            int32_t* d_decisions, int64_t* d_metrics, int32_t* d_trace);

/* ---- RL state / reward shaping on the device snapshot ring (SURVEY.md §8f rank 1) -------------------------------
 * Batched, device-resident forms of the reference's CIM example shaping (examples/cim/rl/env_sampler.py:15-36, 66-80),
 * which issue one snapshot_list query per decision / per reward from Python.  All pointers are device pointers; work is
 * enqueued on the handle's stream and not synchronised.
 *
 * State of replica i, for its decision row d (MARO_DEC_*; rows that are not MARO_STATUS_DECISION give zeros):
 *   ticks  = [max(0, d.tick - rt) for rt in range(look_back - 1)]              (used as frame indices, like the example)
 *   ports  = [d.port] + future_stop_list of d.vessel in the snapshot of frame d.tick
 *   state  = concat(ports snapshot [ticks : ports : port_attrs], vessels snapshot [d.tick : d.vessel : vessel_attrs])
 * as float64, tick -> port -> attr order, zeros for frames the ring no longer holds (np_backend.pyx:536-549).
 * out: [n_replicas][maro_cim_rl_state_dim()] doubles.  Attribute ids come from maro_cim_attr_id (single-slot only). */
int32_t maro_cim_rl_state_dim(MaroCimEnv* env, int32_t look_back, int32_t n_port_attrs, int32_t n_vessel_attrs);
int maro_cim_rl_state_device(MaroCimEnv* env, const int32_t* d_decisions, int32_t look_back, const int32_t* port_attrs,
                             int32_t n_port_attrs, const int32_t* vessel_attrs, int32_t n_vessel_attrs, double* d_out);
/* the same state rounded to float32 (what the example's networks take: torch.from_numpy(states).float()), written straight into
 * the caller's [n_replicas][dim] float buffer — saves the conversion launch inside a collection loop */
int maro_cim_rl_state_f32_device(MaroCimEnv* env, const int32_t* d_decisions, int32_t look_back, const int32_t* port_attrs,
                                 int32_t n_port_attrs, const int32_t* vessel_attrs, int32_t n_vessel_attrs, float* d_out);
/* Action translation (env_sampler.py:38-64) for every replica: model action index m (into d_action_space, n doubles; the
 * example uses [(i - 10) / 10 for i in range(21)]) and the decision row -> action row {vessel, port, quantity, type}:
 *   m < n / 2:  LOAD       min(round(|space[m]| * scope.load), vessel.remaining_space if finite_vessel_space)
 *   else:       DISCHARGE  plan = |space[m]| * (scope.discharge + early) - early, early = vessel.early_discharge if
 *               has_early_discharge else 0; round(plan) if plan > 0 else round(|space[m]| * scope.discharge)
 * with Python's round (half to even); the vessel attributes are read from the decision's snapshot like the example does.
 * out: [n_replicas][max_actions][4] int32 (row 0 written), directly usable as the `actions` of maro_cim_step_device. */
int maro_cim_rl_action_device(MaroCimEnv* env, const int32_t* d_decisions, const int32_t* d_model_actions,
                              const double* d_action_space, int32_t n_action_space, int32_t finite_vessel_space,
                              int32_t has_early_discharge, int32_t* d_actions);
/* The same translation with the bookkeeping a collection loop otherwise spends launches on (each pointer optional): the policy's
 * output taken as int64 (torch argmax) or int32, the index used recorded as int32 [n_replicas], and the previous step's metrics
 * [n_replicas][3] folded into a running maximum — the three CIM metrics are non-negative running totals and a replica stepped past
 * its DONE row reports zeros, so the maximum over an episode is the DONE row's value. */
int maro_cim_rl_action_ex_device(MaroCimEnv* env, const int32_t* d_decisions, const void* d_model_actions, int32_t model_actions_are_i64,
                                 int32_t* d_model_actions_record, const int64_t* d_metrics_in, int64_t* d_metrics_final,
                                 const double* d_action_space, int32_t n_action_space, int32_t finite_vessel_space,
                                 int32_t has_early_discharge, int32_t* d_actions);
/* Reward of replica i for the action it took at tick d_ticks[i] on port d_ports[i] (env_sampler.py:66-80):
 *   float32(fulfillment_factor * sum_k decay[k] * fulfillment[tick+1+k, port]
 *           - shortage_factor * sum_k decay[k] * shortage[tick+1+k, port]),   k = 0 .. time_window-1,
 * d_decay = [time_decay ** k] (time_window doubles on the device).  out: [n_replicas] float32. */
int maro_cim_rl_reward_device(MaroCimEnv* env, const int32_t* d_ticks, const int32_t* d_ports, const double* d_decay,
                              int32_t time_window, double fulfillment_factor, double shortage_factor, float* d_out);
/* The same for a whole trajectory in one launch: d_ticks / d_ports / d_out are [n_rows][n_replicas] (row = rollout step;
 * a negative tick yields reward 0) — the reference computes them one Python call per cached transition
 * (maro/rl/rollout/env_sampler.py:396-402, 500-506). */
int maro_cim_rl_reward_batch_device(MaroCimEnv* env, const int32_t* d_ticks, const int32_t* d_ports, int32_t n_rows,
                                    const double* d_decay, int32_t time_window, double fulfillment_factor,
                                    double shortage_factor, float* d_out);


/* ================================================================================================
 * citi_bike scenario (SURVEY.md §8 row a20): same call shapes as the CIM entry points.
 * Static tables come from maro_b200.scenarios.citi_bike.data.build_bike_topology(), which restates
 * maro/data_lib/binary_reader.py (trace format + ItemTickPicker), citi_bike/business_engine.py:218-396 and
 * decision_strategy.py:385-397.
 * ============================================================================================== */
#define MARO_BIKE_MAX_FILTERS 4
enum { MARO_BIKE_FILTER_DISTANCE = 0, MARO_BIKE_FILTER_REQUIREMENTS = 1, MARO_BIKE_FILTER_TRIP_WINDOW = 2 };
typedef struct MaroBikeTopology {
    int32_t n_stations, n_days;
    int32_t max_tick;            /* start_tick + durations                                            */
    int32_t resolution;          /* decision.resolution (decision_strategy.py:218-227)                */
    int32_t extra_cost_mode;     /* 0 source, 1 target, 2 target_neighbors                            */
    uint32_t transfer_seed;      /* np.random.seed() of the transfer_time stream (:213-216)           */
    double time_mean, time_std;  /* effective_time_mean / _std                                        */
    double supply_ratio, demand_ratio, scope_low, scope_high;
    const int32_t* station_bikes;    /* [S] initial bikes                                             */
    const int32_t* station_capacity; /* [S]                                                           */
    const int32_t* station_id;       /* [S]                                                           */
    const int32_t* nbr_offset;       /* [S+1] neighbours sorted by distance (distance != 0)           */
    const int32_t* nbr_idx;
    const int32_t* trip_offset;      /* [max_tick+1] trips of tick t = [offset[t], offset[t+1])       */
    const int32_t* trip_src;
    const int32_t* trip_dst;
    const int32_t* trip_dur;         /* ticks until the bike is returned                              */
    const int32_t* day_of_tick;      /* [max_tick] row of day_feat                                    */
    const int32_t* day_feat;         /* [n_days][4] weekday, holiday, weather, temperature            */
    /* decision.action_scope.filters, applied in order to the neighbour scope (decision_strategy.py:15-163, 282-283):
     * type 0 "distance" (the `num` nearest neighbours), 1 "requirements" (the `num` largest scope values), 2 "trip_window"
     * (the `num` neighbours with the fewest / most trips over the latest `windows` snapshot frames, per-frame cache incl.) */
    int32_t n_filters;
    int32_t filter_type[MARO_BIKE_MAX_FILTERS], filter_num[MARO_BIKE_MAX_FILTERS], filter_windows[MARO_BIKE_MAX_FILTERS];
} MaroBikeTopology;

/* Decision row: MARO_BIKE_DEC_HEAD int32 header + 2 * n_stations words of (station, scope) pairs in ascending
 * station order (DecisionEvent, citi_bike/common.py:62-127; action_scope dict of decision_strategy.py:253-293). */
enum {
    MARO_BIKE_DEC_TICK = 0,
    MARO_BIKE_DEC_STATION = 1,
    MARO_BIKE_DEC_FRAME_INDEX = 2,
    MARO_BIKE_DEC_TYPE = 3,    /* 0 = Supply, 1 = Demand */
    MARO_BIKE_DEC_N_SCOPE = 4,
    MARO_BIKE_DEC_STATUS = 6,  /* MARO_STATUS_*           */
    MARO_BIKE_DEC_STEP = 7,
    MARO_BIKE_DEC_HEAD = 8
};
/* Action row: 4 int32 {from_station_idx, to_station_idx, number, 0} (citi_bike/common.py:130-150).
 * Metrics row: 3 int64 {trip_requirements, bike_shortage, operation_number} (business_engine.py:211-227). */
enum { MARO_BIKE_NODE_STATIONS = 0, MARO_BIKE_NODE_MATRICES = 1 };

typedef struct MaroBikeEnv MaroBikeEnv;

int maro_bike_create(const MaroBikeTopology* topo, const MaroCimConfig* cfg, MaroBikeEnv** out);
int maro_bike_destroy(MaroBikeEnv* env);
int maro_bike_set_stream(MaroBikeEnv* env, void* cuda_stream, int32_t external);
int32_t maro_bike_decision_words(MaroBikeEnv* env);
/* decisions [B][decision_words] int32, metrics [B][3] int64, actions [B][max_actions][4] int32 */
int maro_bike_step(MaroBikeEnv* env, const uint8_t* active, const int32_t* actions, const int32_t* n_actions,
                   int32_t* decisions, int64_t* metrics);
int maro_bike_pinned_buffers(MaroBikeEnv* env, void** actions, void** n_actions, void** active, void** decisions,
                             void** metrics);
int maro_bike_step_pinned(MaroBikeEnv* env, int32_t use_actions, int32_t use_n_actions, int32_t use_active);
int maro_bike_step_device(MaroBikeEnv* env, const uint8_t* d_active, const int32_t* d_actions,
                          const int32_t* d_n_actions, int32_t* d_decisions, int64_t* d_metrics);
/* Fused rollout (like maro_cim_rollout_device): n_steps env-steps per replica in one launch with the greedy top-1 agent of
 * examples/citi_bike/greedy/launcher.py:35-65 as a device callback; d_decisions is in/out; a replica stops at its DONE row. */
int maro_bike_rollout_device(MaroBikeEnv* env, int32_t n_steps, int32_t* d_decisions, int64_t* d_metrics);
/* Env.reset for the replicas selected by mask (NULL = all).  The mask is read during the call; no pinned staging buffer is
 * written. */
int maro_bike_reset(MaroBikeEnv* env, const uint8_t* mask);
/* Per-replica seeds of the transfer_time stream: the reference draws `round(np.random.normal(mean, std))` per action
 * (citi_bike/decision_strategy.py:213-216) from the process-global numpy RandomState, and every env of a VectorEnv is its
 * own process (maro/vector_env/env_process.py:26-67) — `seeds[k]` is the `np.random.seed` of env k.  uint32 [n_replicas];
 * takes effect at each replica's next reset; NULL = every replica uses the topology's transfer_seed. */
int maro_bike_set_transfer_seeds(MaroBikeEnv* env, const uint32_t* seeds);
int maro_bike_query(MaroBikeEnv* env, const int32_t* replicas, int32_t n_replicas, int32_t node_type,
                    const int32_t* frame_indices, int32_t n_frames, const int32_t* nodes, int32_t n_nodes,
                    const int32_t* attrs, int32_t n_attrs, double* out, int64_t* out_per_replica);
int maro_bike_set_query_layout(MaroBikeEnv* env, int32_t layout); /* see maro_cim_set_query_layout */
int maro_bike_save(MaroBikeEnv* env, const char* path, int32_t with_snapshots); /* see maro_cim_save */
int maro_bike_load(MaroBikeEnv* env, const char* path);
int32_t maro_bike_attr_id(MaroBikeEnv* env, int32_t node_type, const char* name);
int32_t maro_bike_attr_slots(MaroBikeEnv* env, int32_t node_type, int32_t attr_id);
int maro_bike_read_frame(MaroBikeEnv* env, int32_t replica, int32_t* out_words, int32_t n_words);
int32_t maro_bike_frame_words(MaroBikeEnv* env);
int maro_bike_ticks(MaroBikeEnv* env, int32_t* out_ticks);
int maro_bike_counters(MaroBikeEnv* env, int64_t* out);
int maro_bike_snapshot_frames(MaroBikeEnv* env, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out);
/* Agent helper for bench.py: examples/citi_bike/greedy/launcher.py:35-65 with top-1 (deterministic). */
int maro_bike_greedy_policy_device(MaroBikeEnv* env, const int32_t* d_decisions, int32_t* d_actions);

/* ================================================================================================
 * vm_scheduling scenario (SURVEY.md §8 row a21): same call shapes again.
 * Static tables come from maro_b200.scenarios.vm_scheduling.data.build_vm_topology(), which restates
 * vm_scheduling/business_engine.py:131-440 (config / hierarchy), :449-493 (request stream), cpu_reader.py:9-77 and the
 * utilisation-series semantics of virtual_machine.py:73-90.
 * ============================================================================================== */
typedef struct MaroVmTopology {
    int32_t n_pm, n_rack, n_cluster, n_dc, n_zone, n_region, n_pm_types, n_vm;
    int32_t max_tick, delay_duration, buffer_budget, kill_all;
    double ticks_per_hour, max_cpu_over, max_mem_over, max_util_rate, unit_energy_price, pue;
    const int32_t* pm_attr;        /* [n_pm][8] cpu, memory, pm_type, region, zone, dc, cluster, rack           */
    const double* pm_idle_energy;  /* [n_pm]                                                                   */
    const double* pmtype_power;    /* [n_pm_types][3] calibration_parameter, busy_power, idle_power            */
    const int32_t* rack_range;     /* [n_rack][2] pm lo, hi        */
    const int32_t* rack_ids;       /* [n_rack][4] region, zone, dc, cluster */
    const int32_t* cluster_range;  /* [n_cluster][2] rack lo, hi   */
    const int32_t* cluster_ids;    /* [n_cluster][3] region, zone, dc */
    const int32_t* dc_range;       /* [n_dc][2] cluster lo, hi     */
    const int32_t* dc_ids;         /* [n_dc][2] region, zone       */
    const int32_t* zone_range;     /* [n_zone][2] dc lo, hi        */
    const int32_t* zone_ids;       /* [n_zone] region              */
    const int32_t* region_range;   /* [n_region][2] zone lo, hi    */
    const int32_t* vm_attr;        /* [n_vm][8] vm_id, sub_id, deploy_id, request tick, lifetime, category, cores, memory */
    const double* vm_price;        /* [n_vm] unit price per tick (business_engine.py:917-920)                   */
    const int32_t* req_offset;     /* [max_tick+1] requests of tick t = vm indices [offset[t], offset[t+1])     */
    const int32_t* vm_sorted_ids;  /* [n_vm] vm ids ascending      */
    const int32_t* vm_sorted_idx;  /* [n_vm] matching vm indices   */
    const int32_t* util_offset;    /* [n_vm+1] into util_*         */
    const double* util_val;        /* forward-filled readings from the request tick on                         */
    const int32_t* util_has;       /* 1 where the trace holds a reading for that tick                          */
} MaroVmTopology;

/* Decision row: MARO_VM_DEC_HEAD int32 header + n_pm words of valid PM ids, ascending (DecisionEvent,
 * vm_scheduling/common.py:66-120); maro_vm_decision_words() = 12 + n_pm rounded up to a multiple of 4. */
enum {
    MARO_VM_DEC_TICK = 0,
    MARO_VM_DEC_VM_ID = 1,
    MARO_VM_DEC_FRAME_INDEX = 2,
    MARO_VM_DEC_CPU = 3,
    MARO_VM_DEC_MEMORY = 4,
    MARO_VM_DEC_SUB_ID = 5,
    MARO_VM_DEC_STATUS = 6,
    MARO_VM_DEC_STEP = 7,
    MARO_VM_DEC_CATEGORY = 8,
    MARO_VM_DEC_BUFFER_TIME = 9,
    MARO_VM_DEC_N_VALID = 10,
    MARO_VM_DEC_EXT_OFFSET = 11, /* word offset of the extension area: remaining CPU cores (capacity - allocated in the
                                    decision's frame) of valid PM k at row[EXT_OFFSET + k] — what the reference's rule-based
                                    agents fetch with a snapshot query per decision (rule_based_algorithm/best_fit.py:38-44) */
    MARO_VM_DEC_HEAD = 12
};
/* Action row: 4 int32 {vm_id, kind, pm_id | postpone_step, 0}; kind 0 = AllocateAction, 1 = PostponeAction
 * (common.py:9-57).  n_actions = 0 is the reference's empty action list (the pending request is dropped). */
enum { MARO_VM_ACTION_ALLOCATE = 0, MARO_VM_ACTION_POSTPONE = 1 };
/* Metrics row: 16 x 8 bytes (business_engine.py:539-565); float entries are IEEE doubles stored in the int64 slots. */
enum {
    MARO_VM_MET_TOTAL_VM_REQUESTS = 0, MARO_VM_MET_TOTAL_INCOMES_F64 = 1, MARO_VM_MET_ENERGY_COST_F64 = 2,
    MARO_VM_MET_TOTAL_PROFIT_F64 = 3, MARO_VM_MET_TOTAL_ENERGY_F64 = 4, MARO_VM_MET_SUCCESSFUL_ALLOCATION = 5,
    MARO_VM_MET_SUCCESSFUL_COMPLETION = 6, MARO_VM_MET_FAILED_ALLOCATION = 7, MARO_VM_MET_FAILED_COMPLETION = 8,
    MARO_VM_MET_LATENCY_AGENT = 9, MARO_VM_MET_LATENCY_RESOURCE = 10, MARO_VM_MET_OVERSUBSCRIPTIONS = 11,
    MARO_VM_MET_OVERLOAD_PMS = 12, MARO_VM_MET_OVERLOAD_VMS = 13, MARO_VM_METRIC_WORDS = 16
};
enum { MARO_VM_NODE_PMS = 0, MARO_VM_NODE_RACKS = 1, MARO_VM_NODE_CLUSTERS = 2, MARO_VM_NODE_DATA_CENTERS = 3,
       MARO_VM_NODE_ZONES = 4, MARO_VM_NODE_REGIONS = 5 };

typedef struct MaroVmEnv MaroVmEnv;

int maro_vm_create(const MaroVmTopology* topo, const MaroCimConfig* cfg, MaroVmEnv** out);
int maro_vm_destroy(MaroVmEnv* env);
int maro_vm_set_stream(MaroVmEnv* env, void* cuda_stream, int32_t external);
int32_t maro_vm_decision_words(MaroVmEnv* env);
/* decisions [B][decision_words] int32, metrics [B][16] int64, actions [B][max_actions][4] int32 */
int maro_vm_step(MaroVmEnv* env, const uint8_t* active, const int32_t* actions, const int32_t* n_actions,
                 int32_t* decisions, int64_t* metrics);
int maro_vm_step_device(MaroVmEnv* env, const uint8_t* d_active, const int32_t* d_actions, const int32_t* d_n_actions,
                        int32_t* d_decisions, int64_t* d_metrics);
/* zero host-copy variant over the library's pinned staging buffers (see maro_cim_pinned_buffers) */
int maro_vm_pinned_buffers(MaroVmEnv* env, void** actions, void** n_actions, void** active, void** decisions,
                           void** metrics);
int maro_vm_step_pinned(MaroVmEnv* env, int32_t use_actions, int32_t use_n_actions, int32_t use_active);
/* Env.reset for the replicas selected by mask (NULL = all).  The mask is read during the call; no pinned staging buffer is
 * written. */
int maro_vm_reset(MaroVmEnv* env, const uint8_t* mask);
int maro_vm_query(MaroVmEnv* env, const int32_t* replicas, int32_t n_replicas, int32_t node_type,
                  const int32_t* frame_indices, int32_t n_frames, const int32_t* nodes, int32_t n_nodes,
                  const int32_t* attrs, int32_t n_attrs, double* out, int64_t* out_per_replica);
int maro_vm_set_query_layout(MaroVmEnv* env, int32_t layout); /* see maro_cim_set_query_layout */
int maro_vm_save(MaroVmEnv* env, const char* path, int32_t with_snapshots); /* see maro_cim_save */
int maro_vm_load(MaroVmEnv* env, const char* path);
int32_t maro_vm_attr_id(MaroVmEnv* env, int32_t node_type, const char* name);
int32_t maro_vm_attr_slots(MaroVmEnv* env, int32_t node_type, int32_t attr_id);
int maro_vm_read_frame(MaroVmEnv* env, int32_t replica, int32_t* out_words, int32_t n_words);
int32_t maro_vm_frame_words(MaroVmEnv* env);
int maro_vm_ticks(MaroVmEnv* env, int32_t* out_ticks);
int maro_vm_counters(MaroVmEnv* env, int64_t* out);
int maro_vm_snapshot_frames(MaroVmEnv* env, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out);
/* Agent helper for bench.py: best fit (examples/vm_scheduling/rule_based_algorithm/best_fit.py:27-64). */
int maro_vm_best_fit_policy_device(MaroVmEnv* env, const int32_t* d_decisions, int32_t* d_actions);
/* Fused rollouts (device-resident use): n_steps env-steps per launch, the best-fit agent above evaluated between the steps as a
 * device callback; d_decisions / d_metrics carry the last row across launches like maro_cim_rollout_device (a replica stops at
 * its DONE row and keeps the final metrics; the first step after a reset ignores its action, core.py:128). */
int maro_vm_rollout_device(MaroVmEnv* env, int32_t n_steps, int32_t* d_decisions, int64_t* d_metrics);

#ifdef __cplusplus
}
#endif
#endif /* MARO_B200_H */
