// bike_env.cu — kernels + C ABI of the citi_bike scenario (SURVEY.md §8 row a20); device logic in bike_core.cuh.
#include "env_common.cuh"
#include "bike_host.hpp"

// =====================================================================================================
// citi_bike scenario (SURVEY.md §8 row a20)
// =====================================================================================================
struct BikeArgs {
    int32_t* state;
    int32_t* snap;
    int32_t* snap_frame;
    uint32_t* rng;
    const uint32_t* replica_seed;  // [B] per-replica np.random seeds of the transfer_time stream, or nullptr (all replicas share the topology's)
    const int32_t* tables;
    const uint8_t* active;
    const int32_t* actions;
    const int32_t* n_actions;
    int32_t* decisions;
    int64_t* metrics;
    int n_steps;  // > 0: fused rollout — that many env-steps per replica in this launch, greedy top-1 agent as a device callback
};

// greedy top-1 agent (examples/citi_bike/greedy/launcher.py:35-65 with supply_top_k = demand_top_k = 1) on one decision row
__device__ __forceinline__ int4 bike_greedy_row(const int32_t* d) {
    int station = d[1], ns = d[4], best = -1, best_v = 0;
    for (int k = 0; k < ns; k++) {
        int idx = d[8 + 2 * k], v = d[9 + 2 * k];
        if (idx == station) continue;
        if (best < 0 || v > best_v || (v == best_v && idx > best)) { best = idx; best_v = v; }
    }
    return best < 0 ? make_int4(-1, -1, 0, 0) : (d[3] == 0 ? make_int4(station, best, best_v, 0) : make_int4(best, station, best_v, 0));
}

__device__ __forceinline__ BikeReplica make_bike_replica(const BikeShape& s, const BikeArgs& a, int rep, int32_t* st) {
    BikeReplica r;
    r.f = st;
    r.c = st + s.FWp;
    r.q = st + s.FWp + s.CWp;
    r.t = a.tables;
    r.rng = a.rng + (int64_t)rep * s.rng_words;
    r.seed = a.replica_seed ? (int64_t)a.replica_seed[rep] : -1;
    r.snap = a.snap + (int64_t)rep * s.ring_rows * s.FWp;
    r.snap_frame = a.snap_frame + (int64_t)rep * s.ring_rows;
    return r;
}

template <int kWarps, int G, bool kSpread = false>  // kSpread: one replica per warp, see cim_step_kernel
__global__ void __launch_bounds__(kWarps * 32) bike_step_kernel(const __grid_constant__ BikeShape s,
                                                                const __grid_constant__ BikeArgs a) {
    constexpr int kGroups = kSpread ? kWarps : kWarps * 32 / G;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
    if (kSpread && (threadIdx.x & 31) >= G) return;
    const int gid = kSpread ? threadIdx.x >> 5 : threadIdx.x / G;
    const Grp<G> g(threadIdx.x & 31);
    int32_t* st = reinterpret_cast<int32_t*>(smem_raw + 256) + (size_t)gid * s.SW;
    uint64_t* bar = bars + gid;
    if (g.lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
    }
    g.sync();
    uint32_t phase = 0;
    const uint32_t bytes = (uint32_t)s.SW * 4u;
    for (int rep = blockIdx.x * kGroups + gid; rep < s.n_replicas; rep += gridDim.x * kGroups) {
        if (a.active && !a.active[rep]) {
            if (g.lane == 0) a.decisions[(int64_t)rep * s.DW + 6] = MARO_STATUS_INACTIVE;
            continue;
        }
        int32_t* gstate = a.state + (int64_t)rep * s.SW;
        if (g.lane == 0) {
            fence_proxy_async();
            mbar_expect_tx(bar, bytes);
            bulk_g2s(st, gstate, bytes, bar);
        }
        while (!mbar_try_wait(bar, phase)) {}
        phase ^= 1u;
        BikeReplica r = make_bike_replica(s, a, rep, st);
        if (a.n_steps > 0) {
            // ---- fused rollout: the block stays in shared memory for n_steps env-steps; the decision row lives in a
            // per-group shared-memory slot between the steps and feeds the agent; stops at the replica's DONE row
            const int slot_bytes = (s.DW * 4 + 24 + 15) & ~15;
            int32_t* dslot = reinterpret_cast<int32_t*>(smem_raw + 256 + (size_t)kGroups * s.SW * 4 + (size_t)gid * slot_bytes);
            int64_t* mslot = reinterpret_cast<int64_t*>(dslot + ((s.DW + 1) & ~1));
            int32_t* gdec = a.decisions + (int64_t)rep * s.DW;
            for (int i = g.lane; i < s.DW; i += G) dslot[i] = gdec[i];
            g.sync();
            for (int k = 0; k < a.n_steps; k++) {
                Act4 act = {0, 0, 0, 0};
                if (g.lane == 0) {
                    int4 o = bike_greedy_row(dslot);
                    act.v = o.x; act.p = o.y; act.qty = o.z; act.type = o.w;
                }
                bike_replica_step<G>(s, g, r, act, 1, dslot, mslot);
                g.sync();
                if (dslot[6] != MARO_STATUS_DECISION) break;  // DONE (final metrics stay in the slot) / FINISHED / error
            }
            for (int i = g.lane; i < s.DW; i += G) gdec[i] = dslot[i];
            if (g.lane < 3) a.metrics[(int64_t)rep * 3 + g.lane] = mslot[g.lane];
        } else {
        const int n_act = a.actions ? (a.n_actions ? min(max(a.n_actions[rep], 0), min(s.max_actions, G)) : 1) : 0;
        Act4 act = {0, 0, 0, 0};
        if (g.lane < n_act) {
            int4 v = reinterpret_cast<const int4*>(a.actions + (int64_t)rep * s.max_actions * 4)[g.lane];
            act.v = v.x; act.p = v.y; act.qty = v.z; act.type = v.w;
        }
        bike_replica_step<G>(s, g, r, act, n_act, a.decisions + (int64_t)rep * s.DW, a.metrics + (int64_t)rep * 3);
        }
        const int4* src4 = reinterpret_cast<const int4*>(st);
        int4* dst4 = reinterpret_cast<int4*>(gstate);
        for (int i = g.lane; i < s.SW / 4; i += G) dst4[i] = src4[i];
        g.sync();
    }
}

__global__ void bike_reset_kernel(const __grid_constant__ BikeShape s, const __grid_constant__ BikeArgs a) {
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const Grp<32> g(threadIdx.x & 31);
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    for (int rep = warp_global; rep < s.n_replicas; rep += n_warps) {
        if (a.active && !a.active[rep]) continue;
        BikeReplica r = make_bike_replica(s, a, rep, a.state + (int64_t)rep * s.SW);
        bike_replica_reset<32>(s, g, r);
    }
}

// greedy top-1 agent (examples/citi_bike/greedy/launcher.py:35-65 with supply_top_k = demand_top_k = 1)
__global__ void bike_greedy_kernel(const int32_t* __restrict__ dec, int32_t* __restrict__ act, int n, int dw, int max_actions) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    *reinterpret_cast<int4*>(act + (int64_t)i * max_actions * 4) = bike_greedy_row(dec + (int64_t)i * dw);
}

struct MaroBikeEnv : EnvCommon {
    BikeShape s;
    int warps_per_cta = 1, lanes = 8, grid = 0;
    bool spread = false;
    size_t smem_bytes = 0;
    int32_t* d_tables = nullptr;
    uint32_t* d_rng = nullptr;
    uint32_t* d_replica_seed = nullptr;
    std::vector<int32_t> h_tables;
};

static BikeArgs bike_base_args(MaroBikeEnv* e) {
    BikeArgs a;
    memset(&a, 0, sizeof(a));
    a.state = e->d_state; a.snap = e->d_snap; a.snap_frame = e->d_snap_frame; a.rng = e->d_rng; a.tables = e->d_tables;
    a.replica_seed = e->d_replica_seed;
    return a;
}

template <int W, int G>
static cudaError_t bike_launch_wg(MaroBikeEnv* e, const BikeArgs& a) {
    // fused rollouts keep one decision-row slot per lane group behind the state blocks
    const int groups = (G < 32 && W == 4 && e->spread) ? W : W * 32 / G;
    const size_t smem = e->smem_bytes + (a.n_steps > 0 ? (size_t)groups * ((e->s.DW * 4 + 24 + 15) & ~15) : 0);
    if (G < 32 && W == 4 && e->spread) {
        cudaError_t err = cudaFuncSetAttribute(bike_step_kernel<W, G, (G < 32 && W == 4)>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return err;
        bike_step_kernel<W, G, (G < 32 && W == 4)><<<e->grid, W * 32, smem, e->stream>>>(e->s, a);
        return cudaGetLastError();
    }
    cudaError_t err = cudaFuncSetAttribute(bike_step_kernel<W, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    bike_step_kernel<W, G><<<e->grid, W * 32, smem, e->stream>>>(e->s, a);
    return cudaGetLastError();
}
template <int G>
static cudaError_t bike_launch_g(MaroBikeEnv* e, const BikeArgs& a) {
    switch (e->warps_per_cta) {
        case 1: return bike_launch_wg<1, G>(e, a);
        case 2: return bike_launch_wg<2, G>(e, a);
        case 4: return bike_launch_wg<4, G>(e, a);
        default: return bike_launch_wg<8, G>(e, a);
    }
}
static cudaError_t bike_launch(MaroBikeEnv* e, const BikeArgs& a) {
    switch (e->lanes) {
        case 8: return bike_launch_g<8>(e, a);
        case 16: return bike_launch_g<16>(e, a);
        default: return bike_launch_g<32>(e, a);
    }
}


// inside *_create, after the handle exists: a failing CUDA call frees it before returning
#define CKD(call)                                                                                     \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) { maro_bike_destroy(e); return fail(std::string(#call) + ": " + cudaGetErrorString(e__)); } \
    } while (0)
extern "C" int maro_bike_destroy(MaroBikeEnv* e);
extern "C" {

int maro_bike_destroy(MaroBikeEnv* e) {
    if (!e) return 0;
    cudaSetDevice(e->device);
    cudaFree(e->d_tables); cudaFree(e->d_rng); cudaFree(e->d_replica_seed);
    common_free(e);
    delete e;
    return 0;
}

int maro_bike_reset(MaroBikeEnv* e, const uint8_t* mask) {
    if (!e) return fail("null handle");
    CK(cudaSetDevice(e->device));
    BikeArgs a = bike_base_args(e);
    if (mask && common_stage_mask(e, mask, &a.active)) return 1;
    int threads = 128, blocks = std::min((e->B * 32 + threads - 1) / threads, e->n_sm * 16);
    bike_reset_kernel<<<blocks, threads, 0, e->stream>>>(e->s, a);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

int maro_bike_create(const MaroBikeTopology* topo, const MaroCimConfig* cfg, MaroBikeEnv** out) {
    if (!topo || !cfg || !out || cfg->n_replicas < 1) return fail("maro_bike_create: bad arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("maro_bike_create: no CUDA device — this library has no CPU path");
    if (cfg->device < 0 || cfg->device >= ndev) return fail("maro_bike_create: bad device ordinal");
    CK(cudaSetDevice(cfg->device));
    MaroBikeEnv* e = new MaroBikeEnv();
    e->device = cfg->device;
    e->B = cfg->n_replicas;
    BikeShape& s = e->s;
    if (int rc = bike_compute_shape_and_tables(*topo, cfg, s, e->h_tables)) {
        delete e;
        return fail(rc == 2 ? "maro_bike_create: a 'distance' action-scope filter behind a filter that drops neighbours raises KeyError in the "
                              "reference (decision_strategy.py:45-48); put it first"
                            : "maro_bike_create: bad topology (1..255 stations, durations > 0, at most 4 action-scope filters)");
    }
    e->n_node_types = 2;
    static const char* an[] = {"bikes", "capacity", "extra_cost", "failed_return", "fulfillment", "holiday", "id", "min_bikes",
                               "shortage", "temperature", "transfer_cost", "trip_requirement", "weather", "weekday"};
    for (int a = 0; a < BA_COUNT; a++) e->attrs[0].push_back({an[a], a * s.S, 1, 0, s.S});
    e->attrs[1].push_back({"trips_adj", BA_COUNT * s.S, s.S * s.S, 0, 1});
    cudaDeviceProp prop;
    CKD(cudaGetDeviceProperties(&prop, e->device));
    e->lanes = bike_lanes_per_replica(s);
    const int gpw = 32 / e->lanes;
    const size_t per_warp = (size_t)s.SW * 4 * gpw;
    const size_t max_smem = prop.sharedMemPerBlockOptin, sm_smem = prop.sharedMemPerMultiprocessor;
    if (256 + per_warp > max_smem) { delete e; return fail("maro_bike_create: replica state does not fit in shared memory"); }
    int w = 1, best = 0;
    for (int cand = 8; cand >= 1; cand >>= 1) {
        size_t cta = 256 + per_warp * cand;
        if (cta > max_smem) continue;
        int blocks = (int)std::min<size_t>(sm_smem / (cta + 1024), (size_t)(32 / cand));
        if (blocks * cand > best) { best = blocks * cand; w = cand; }
    }
    while (w > 1 && (e->B + w * gpw - 1) / (w * gpw) < prop.multiProcessorCount) w >>= 1;
    e->warps_per_cta = w;
    e->smem_bytes = 256 + per_warp * w;
    int ctas_needed = (e->B + w * gpw - 1) / (w * gpw);
    int resident = std::max<int>(1, (int)std::min<size_t>(32 / w, sm_smem / (e->smem_bytes + 1024)));
    e->grid = std::min(ctas_needed, prop.multiProcessorCount * resident);
    {   // the tick chain runs on each group's leader lane: packed groups serialise their leaders, so spread when possible
        const char* sp = getenv("MARO_B200_SPREAD");
        const bool want_spread = sp ? atoi(sp) != 0 : e->B <= prop.multiProcessorCount * 128;  // the leader-lane chain gains from a warp of its own
        if (gpw > 1 && want_spread && 256 + (size_t)s.SW * 4 * 4 <= max_smem) {
            e->spread = true;
            e->warps_per_cta = 4;
            e->smem_bytes = 256 + (size_t)s.SW * 4 * 4;
            e->grid = (e->B + 3) / 4;
        }
    }
    e->ring_rows = s.ring_rows; e->FW = s.FW; e->FWp = s.FWp; e->SW = s.SW;
    e->off_tick = s.FWp + BC_TICK; e->off_counters = s.FWp + BC_NSTEPS_LO;
    e->dec_words = s.DW; e->max_actions = s.max_actions;
    if (common_alloc(e)) { maro_bike_destroy(e); return 1; }
    CKD(cudaMalloc(&e->d_tables, e->h_tables.size() * 4));
    CKD(cudaMemcpy(e->d_tables, e->h_tables.data(), e->h_tables.size() * 4, cudaMemcpyHostToDevice));
    CKD(cudaMalloc(&e->d_rng, (size_t)e->B * s.rng_words * 4));
    e->scenario_id = 2;
    e->ckpt_extra = {{"rng", (void**)&e->d_rng, (size_t)e->B * s.rng_words * 4}};
    *out = e;
    int rc = maro_bike_reset(e, nullptr);
    if (rc) { maro_bike_destroy(e); *out = nullptr; return rc; }
    return 0;
}

int maro_bike_set_stream(MaroBikeEnv* e, void* cuda_stream, int32_t external) {
    if (!e) return fail("null handle");
    e->stream = external ? (cudaStream_t)cuda_stream : e->own_stream;
    return 0;
}
/* Per-replica seeds of the transfer_time stream (np.random.seed(k) in the process of env k); they take effect at the next
   reset of each replica.  NULL returns to the topology's single transfer_seed. */
int maro_bike_set_transfer_seeds(MaroBikeEnv* e, const uint32_t* seeds) {
    if (!e) return fail("null handle");
    CK(cudaSetDevice(e->device));
    if (!seeds) {
        CK(cudaStreamSynchronize(e->stream));
        cudaFree(e->d_replica_seed);
        e->d_replica_seed = nullptr;
        return 0;
    }
    if (!e->d_replica_seed) CK(cudaMalloc(&e->d_replica_seed, (size_t)e->B * 4));
    CK(cudaMemcpyAsync(e->d_replica_seed, seeds, (size_t)e->B * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}
int32_t maro_bike_decision_words(MaroBikeEnv* e) { return e ? e->s.DW : -1; }
int32_t maro_bike_frame_words(MaroBikeEnv* e) { return e ? e->s.FW : -1; }

int maro_bike_step_device(MaroBikeEnv* e, const uint8_t* d_active, const int32_t* d_actions, const int32_t* d_n_actions,
                          int32_t* d_decisions, int64_t* d_metrics) {
    if (!e || !d_decisions || !d_metrics) return fail("maro_bike_step_device: bad arguments");
    CK(cudaSetDevice(e->device));
    BikeArgs a = bike_base_args(e);
    a.active = d_active; a.actions = d_actions; a.n_actions = d_n_actions; a.decisions = d_decisions; a.metrics = d_metrics;
    CK(bike_launch(e, a));
    return 0;
}
int maro_bike_step(MaroBikeEnv* e, const uint8_t* active, const int32_t* actions, const int32_t* n_actions, int32_t* decisions,
                   int64_t* metrics) {
    if (!e || !decisions || !metrics) return fail("maro_bike_step: bad arguments");
    CK(cudaSetDevice(e->device));
    return common_host_step(e, active, actions, n_actions, decisions, metrics,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_bike_step_device(e, a, ac, na, d, m);
                            });
}
int maro_bike_pinned_buffers(MaroBikeEnv* e, void** actions, void** n_actions, void** active, void** decisions, void** metrics) {
    return common_pinned_buffers(e, actions, n_actions, active, decisions, metrics);
}
int maro_bike_step_pinned(MaroBikeEnv* e, int32_t use_actions, int32_t use_n_actions, int32_t use_active) {
    if (!e) return fail("maro_bike_step_pinned: null handle");
    CK(cudaSetDevice(e->device));
    const uint8_t* f = reinterpret_cast<const uint8_t*>(1);
    return common_host_step(e, use_active ? f : nullptr, use_actions ? reinterpret_cast<const int32_t*>(f) : nullptr,
                            use_n_actions ? reinterpret_cast<const int32_t*>(f) : nullptr, nullptr, nullptr,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_bike_step_device(e, a, ac, na, d, m);
                            }, true);
}
int maro_bike_query(MaroBikeEnv* e, const int32_t* replicas, int32_t n_replicas, int32_t node_type, const int32_t* frame_indices,
                    int32_t n_frames, const int32_t* nodes, int32_t n_nodes, const int32_t* attrs, int32_t n_attrs, double* out,
                    int64_t* out_per_replica) {
    if (!out) return fail("maro_bike_query: null output");
    return query_impl(e, replicas, n_replicas, node_type, frame_indices, n_frames, nodes, n_nodes, attrs, n_attrs, nullptr, out, out_per_replica);
}
int maro_bike_save(MaroBikeEnv* e, const char* path, int32_t with_snapshots) { return common_save(e, path, with_snapshots); }
int maro_bike_load(MaroBikeEnv* e, const char* path) { return common_load(e, path); }
int maro_bike_set_query_layout(MaroBikeEnv* e, int32_t layout) { return common_set_query_layout(e, layout); }
int32_t maro_bike_attr_id(MaroBikeEnv* e, int32_t node_type, const char* name) { return common_attr_id(e, node_type, name); }
int32_t maro_bike_attr_slots(MaroBikeEnv* e, int32_t node_type, int32_t attr_id) { return common_attr_slots(e, node_type, attr_id); }
int maro_bike_read_frame(MaroBikeEnv* e, int32_t replica, int32_t* out_words, int32_t n_words) { return common_read_frame(e, replica, out_words, n_words); }
int maro_bike_ticks(MaroBikeEnv* e, int32_t* out_ticks) { return common_ticks(e, out_ticks); }
int maro_bike_counters(MaroBikeEnv* e, int64_t* out) { return common_counters(e, out); }
int maro_bike_snapshot_frames(MaroBikeEnv* e, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out) {
    return common_snapshot_frames(e, replica, out, cap, n_out);
}
/* n_steps fused env-steps per replica in ONE launch (the replica block stays in shared memory), greedy top-1 agent evaluated on
   the device between the steps; d_decisions is in/out (the rows the previous call returned feed the first action). */
int maro_bike_rollout_device(MaroBikeEnv* e, int32_t n_steps, int32_t* d_decisions, int64_t* d_metrics) {
    if (!e || !d_decisions || !d_metrics || n_steps < 1) return fail("maro_bike_rollout_device: bad arguments");
    CK(cudaSetDevice(e->device));
    BikeArgs a = bike_base_args(e);
    a.decisions = d_decisions; a.metrics = d_metrics; a.n_steps = n_steps;
    CK(bike_launch(e, a));
    return 0;
}

int maro_bike_greedy_policy_device(MaroBikeEnv* e, const int32_t* d_decisions, int32_t* d_actions) {
    if (!e || !d_decisions || !d_actions) return fail("maro_bike_greedy_policy_device: bad arguments");
    CK(cudaSetDevice(e->device));
    int threads = 256, blocks = (e->B + threads - 1) / threads;
    bike_greedy_kernel<<<blocks, threads, 0, e->stream>>>(d_decisions, d_actions, e->B, e->s.DW, e->s.max_actions);
    CK(cudaGetLastError());
    return 0;
}

}  // extern "C"

