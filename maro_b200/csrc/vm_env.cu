// vm_env.cu — kernels + C ABI of the vm_scheduling scenario (SURVEY.md §8 row a21); device logic in vm_core.cuh.
#include "env_common.cuh"
#include "vm_host.hpp"

// =====================================================================================================
// vm_scheduling scenario (SURVEY.md §8 row a21)
// =====================================================================================================
struct VmArgs {
    int32_t* state;
    int32_t* snap;
    int32_t* snap_frame;
    const int32_t* tables;
    const uint8_t* active;
    const int32_t* actions;
    const int32_t* n_actions;
    int32_t* decisions;
    int64_t* metrics;
    int n_steps;  // vm_rollout_kernel: env-steps fused into the launch
};

// One warp = one replica; the replica block stays in global memory (L2), see vm_core.cuh.
template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32) vm_step_kernel(const __grid_constant__ VmShape s, const __grid_constant__ VmArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int wid = threadIdx.x >> 5;
    const Grp<32> g(threadIdx.x & 31);
    double* scratch = reinterpret_cast<double*>(smem_raw) + (size_t)wid * 2 * s.N;
    for (int rep = blockIdx.x * kWarps + wid; rep < s.n_replicas; rep += gridDim.x * kWarps) {
        if (a.active && !a.active[rep]) {
            if (g.lane == 0) a.decisions[(int64_t)rep * s.DW + MARO_VM_DEC_STATUS] = MARO_STATUS_INACTIVE;
            continue;
        }
        VmReplica r = vm_replica_at(s, a.state, a.tables, a.snap, a.snap_frame, (size_t)rep);
        const int n_act = a.actions ? (a.n_actions ? min(max(a.n_actions[rep], 0), s.max_actions) : 1) : 0;
        vm_replica_step<32>(s, g, r, a.actions ? a.actions + (int64_t)rep * s.max_actions * 4 : nullptr, n_act,
                            a.decisions + (int64_t)rep * s.DW, a.metrics + (int64_t)rep * MARO_VM_METRIC_WORDS, scratch);
    }
}

// Fused rollouts: `n_steps` env-steps per launch with the rule-based best-fit agent of the reference's example as a device callback
// (examples/vm_scheduling/rule_based_algorithm/best_fit.py:27-64, metric "remaining_cpu_cores": among the valid PMs the one with
// the fewest remaining cores, first minimum wins — read from the decision row's remaining-cores extension).  The decision row, the
// metrics and the action stay in shared memory between the steps; the replica's lines of the state block stay in this SM's L1.
// per warp: scratch (2 N doubles, padded to 16 B) | metrics slot | action row | decision row
__host__ __device__ inline size_t vm_rollout_scratch_bytes(int n_pm) { return ((size_t)2 * n_pm * sizeof(double) + 15) & ~(size_t)15; }
__host__ __device__ inline size_t vm_rollout_warp_bytes(int n_pm, int dec_words) {
    return vm_rollout_scratch_bytes(n_pm) + MARO_VM_METRIC_WORDS * 8 + 16 + (((size_t)dec_words * 4 + 15) & ~(size_t)15);
}
template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32) vm_rollout_kernel(const __grid_constant__ VmShape s, const __grid_constant__ VmArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int wid = threadIdx.x >> 5;
    const Grp<32> g(threadIdx.x & 31);
    const size_t scratch_bytes = vm_rollout_scratch_bytes(s.N), per_warp = vm_rollout_warp_bytes(s.N, s.DW);
    unsigned char* mine = smem_raw + (size_t)wid * per_warp;
    double* scratch = reinterpret_cast<double*>(mine);
    int64_t* mslot = reinterpret_cast<int64_t*>(mine + scratch_bytes);
    int32_t* aslot = reinterpret_cast<int32_t*>(mslot + MARO_VM_METRIC_WORDS);
    int32_t* dslot = aslot + 4;
    for (int rep = blockIdx.x * kWarps + wid; rep < s.n_replicas; rep += gridDim.x * kWarps) {
        VmReplica r = vm_replica_at(s, a.state, a.tables, a.snap, a.snap_frame, (size_t)rep);
        int32_t* gdec = a.decisions + (int64_t)rep * s.DW;
        int64_t* gmet = a.metrics + (int64_t)rep * MARO_VM_METRIC_WORDS;
        for (int i = g.lane; i < s.DW; i += 32) dslot[i] = gdec[i];  // the decision the previous launch returned (feeds the agent)
        if (g.lane < MARO_VM_METRIC_WORDS) mslot[g.lane] = gmet[g.lane];
        g.sync();
        for (int k = 0; k < a.n_steps; k++) {
            const int n = dslot[MARO_VM_DEC_STATUS] == MARO_STATUS_DECISION ? dslot[MARO_VM_DEC_N_VALID] : 0;
            const int ext = dslot[MARO_VM_DEC_EXT_OFFSET];
            long long best = 0x7fffffffffffffffLL;
            for (int j = g.lane; j < n; j += 32) {
                const long long key = (long long)dslot[ext + j] * 4294967296LL + j;
                best = key < best ? key : best;
            }
            for (int o = 16; o > 0; o >>= 1) {
                const long long other = __shfl_xor_sync(0xffffffffu, best, o);
                best = other < best ? other : best;
            }
            if (g.lane == 0) {
                const int4 row = n > 0 ? make_int4(dslot[MARO_VM_DEC_VM_ID], MARO_VM_ACTION_ALLOCATE, dslot[MARO_VM_DEC_HEAD + (int)(best & 0xffffffffLL)], 0)
                                       : make_int4(-1, -1, 0, 0);
                *reinterpret_cast<int4*>(aslot) = row;
            }
            g.sync();
            vm_replica_step<32>(s, g, r, aslot, 1, dslot, mslot, scratch);
            g.sync();
            if (dslot[MARO_VM_DEC_STATUS] != MARO_STATUS_DECISION) break;  // DONE (final metrics stay in the slot) / FINISHED / error
        }
        for (int i = g.lane; i < s.DW; i += 32) gdec[i] = dslot[i];
        if (g.lane < MARO_VM_METRIC_WORDS) gmet[g.lane] = mslot[g.lane];
        g.sync();
    }
}

__global__ void vm_reset_kernel(const __grid_constant__ VmShape s, const __grid_constant__ VmArgs a, int init_ring) {
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const Grp<32> g(threadIdx.x & 31);
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    for (int rep = warp_global; rep < s.n_replicas; rep += n_warps) {
        if (a.active && !a.active[rep]) continue;
        VmReplica r = vm_replica_at(s, a.state, a.tables, a.snap, a.snap_frame, (size_t)rep);
        vm_replica_reset<32>(s, g, r, init_ring != 0);
    }
}

// best fit (examples/vm_scheduling/rule_based_algorithm/best_fit.py:27-64, metric "remaining_cpu_cores"): among the valid
// PMs the one with the fewest remaining cores in the decision's snapshot (= the live frame), first minimum wins.
__global__ void vm_best_fit_kernel(const __grid_constant__ VmShape s, const int32_t* __restrict__ state,
                                   const int32_t* __restrict__ dec, int32_t* __restrict__ act) {
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    for (int rep = warp_global; rep < s.n_replicas; rep += n_warps) {
        const int32_t* d = dec + (int64_t)rep * s.DW;
        const int32_t* f = state + (int64_t)rep * s.SW;
        const int n = d[MARO_VM_DEC_STATUS] == MARO_STATUS_DECISION ? d[MARO_VM_DEC_N_VALID] : 0;
        long long best = 0x7fffffffffffffffLL;
        for (int k = lane; k < n; k += 32) {
            int p = d[MARO_VM_DEC_HEAD + k];
            long long key = (long long)(f[VPA_CPU_CAP * s.N + p] - f[VPA_CPU_ALLOC * s.N + p]) * 4294967296LL + k;
            best = key < best ? key : best;
        }
        for (int o = 16; o > 0; o >>= 1) {
            long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other < best ? other : best;
        }
        if (lane == 0) {
            int4 out = n > 0 ? make_int4(d[MARO_VM_DEC_VM_ID], MARO_VM_ACTION_ALLOCATE, d[MARO_VM_DEC_HEAD + (int)(best & 0xffffffffLL)], 0)
                             : make_int4(-1, -1, 0, 0);
            *reinterpret_cast<int4*>(act + (int64_t)rep * s.max_actions * 4) = out;
        }
    }
}

struct MaroVmEnv : EnvCommon {
    VmShape s;
    int warps_per_cta = 4, grid = 0;
    size_t smem_bytes = 0;
    int32_t* d_tables = nullptr;
    std::vector<int32_t> h_tables;
};

static VmArgs vm_base_args(MaroVmEnv* e) {
    VmArgs a;
    memset(&a, 0, sizeof(a));
    a.state = e->d_state; a.snap = e->d_snap; a.snap_frame = e->d_snap_frame; a.tables = e->d_tables;
    return a;
}

static cudaError_t vm_launch(MaroVmEnv* e, const VmArgs& a) {
    switch (e->warps_per_cta) {
        case 1: vm_step_kernel<1><<<e->grid, 32, e->smem_bytes, e->stream>>>(e->s, a); break;
        case 2: vm_step_kernel<2><<<e->grid, 64, e->smem_bytes, e->stream>>>(e->s, a); break;
        default: vm_step_kernel<4><<<e->grid, 128, e->smem_bytes, e->stream>>>(e->s, a); break;
    }
    return cudaGetLastError();
}


// inside *_create, after the handle exists: a failing CUDA call frees it before returning
#define CKD(call)                                                                                     \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) { maro_vm_destroy(e); return fail(std::string(#call) + ": " + cudaGetErrorString(e__)); } \
    } while (0)
extern "C" int maro_vm_destroy(MaroVmEnv* e);
extern "C" {

int maro_vm_destroy(MaroVmEnv* e) {
    if (!e) return 0;
    cudaSetDevice(e->device);
    cudaFree(e->d_tables);
    common_free(e);
    delete e;
    return 0;
}

static int vm_reset_impl(MaroVmEnv* e, const uint8_t* mask, int init_ring) {
    if (!e) return fail("null handle");
    CK(cudaSetDevice(e->device));
    VmArgs a = vm_base_args(e);
    if (mask && common_stage_mask(e, mask, &a.active)) return 1;
    int threads = 128, blocks = std::min((e->B * 32 + threads - 1) / threads, e->n_sm * 16);
    vm_reset_kernel<<<blocks, threads, 0, e->stream>>>(e->s, a, init_ring);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}
int maro_vm_reset(MaroVmEnv* e, const uint8_t* mask) { return vm_reset_impl(e, mask, 0); }

int maro_vm_create(const MaroVmTopology* topo, const MaroCimConfig* cfg, MaroVmEnv** out) {
    if (!topo || !cfg || !out || cfg->n_replicas < 1) return fail("maro_vm_create: bad arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("maro_vm_create: no CUDA device — this library has no CPU path");
    if (cfg->device < 0 || cfg->device >= ndev) return fail("maro_vm_create: bad device ordinal");
    CK(cudaSetDevice(cfg->device));
    MaroVmEnv* e = new MaroVmEnv();
    e->device = cfg->device;
    e->B = cfg->n_replicas;
    VmShape& s = e->s;
    std::string why = vm_compute_shape_and_tables(*topo, cfg, s, e->h_tables);
    if (!why.empty()) { delete e; return fail("maro_vm_create: " + why); }
    e->n_node_types = 6;
    static const char* pn[] = {"cluster_id", "cpu_cores_allocated", "cpu_cores_capacity", "cpu_utilization", "data_center_id",
                               "energy_consumption", "id", "memory_allocated", "memory_capacity", "oversubscribable", "pm_type",
                               "rack_id", "region_id", "zone_id"};
    for (int a = 0; a < VPA_COUNT; a++) e->attrs[0].push_back({pn[a], a * s.N, 1, a == VPA_CPU_UTIL || a == VPA_ENERGY, s.N});
    static const char* rn[] = {"cluster_id", "data_center_id", "empty_machine_num", "id", "region_id", "total_machine_num", "zone_id"};
    for (int a = 0; a < 7; a++) e->attrs[1].push_back({rn[a], s.o_rack + a * s.R, 1, 0, s.R});
    static const char* cn[] = {"data_center_id", "empty_machine_num", "id", "region_id", "total_machine_num", "zone_id"};
    for (int a = 0; a < 6; a++) e->attrs[2].push_back({cn[a], s.o_cluster + a * s.C, 1, 0, s.C});
    static const char* dn[] = {"empty_machine_num", "id", "region_id", "total_machine_num", "zone_id"};
    for (int a = 0; a < 5; a++) e->attrs[3].push_back({dn[a], s.o_dc + a * s.D, 1, 0, s.D});
    static const char* zn[] = {"empty_machine_num", "id", "region_id", "total_machine_num"};
    for (int a = 0; a < 4; a++) e->attrs[4].push_back({zn[a], s.o_zone + a * s.Z, 1, 0, s.Z});
    static const char* gn[] = {"empty_machine_num", "id", "total_machine_num"};
    for (int a = 0; a < 3; a++) e->attrs[5].push_back({gn[a], s.o_region + a * s.RG, 1, 0, s.RG});
    cudaDeviceProp prop;
    CKD(cudaGetDeviceProperties(&prop, e->device));
    int w = 4;
    while (w > 1 && (e->B + w - 1) / w < prop.multiProcessorCount) w >>= 1;
    // per-warp scratch of 2 N doubles: fewer warps per CTA for big clusters, then the opt-in shared-memory carve-out
    while (w > 1 && (size_t)w * 2 * s.N * sizeof(double) > 48 * 1024) w >>= 1;
    e->warps_per_cta = w;
    e->smem_bytes = (size_t)w * 2 * s.N * sizeof(double);
    if (e->smem_bytes > 48 * 1024) {
        if (e->smem_bytes > prop.sharedMemPerBlockOptin) { delete e; return fail("maro_vm_create: too many PMs for the per-warp scratch"); }
        CKD(cudaFuncSetAttribute(vm_step_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem_bytes));
    }
    e->grid = std::min((e->B + w - 1) / w, prop.multiProcessorCount * (48 / w));
    e->ring_rows = s.ring_rows; e->FW = s.FW; e->FWp = s.FWp; e->SW = s.SW;
    e->off_tick = s.FWp + VC_TICK; e->off_counters = s.FWp + VC_NSTEPS;
    e->dec_words = s.DW; e->max_actions = s.max_actions; e->met_words = MARO_VM_METRIC_WORDS;
    if (common_alloc(e)) { maro_vm_destroy(e); return 1; }
    CKD(cudaMalloc(&e->d_tables, e->h_tables.size() * 4));
    CKD(cudaMemcpy(e->d_tables, e->h_tables.data(), e->h_tables.size() * 4, cudaMemcpyHostToDevice));
    e->scenario_id = 3;
    *out = e;
    int rc = vm_reset_impl(e, nullptr, 1);
    if (rc) { maro_vm_destroy(e); *out = nullptr; return rc; }
    return 0;
}

int maro_vm_set_stream(MaroVmEnv* e, void* cuda_stream, int32_t external) {
    if (!e) return fail("null handle");
    e->stream = external ? (cudaStream_t)cuda_stream : e->own_stream;
    return 0;
}
int32_t maro_vm_decision_words(MaroVmEnv* e) { return e ? e->s.DW : -1; }
int32_t maro_vm_frame_words(MaroVmEnv* e) { return e ? e->s.FW : -1; }

int maro_vm_step_device(MaroVmEnv* e, const uint8_t* d_active, const int32_t* d_actions, const int32_t* d_n_actions,
                        int32_t* d_decisions, int64_t* d_metrics) {
    if (!e || !d_decisions || !d_metrics) return fail("maro_vm_step_device: bad arguments");
    CK(cudaSetDevice(e->device));
    VmArgs a = vm_base_args(e);
    a.active = d_active; a.actions = d_actions; a.n_actions = d_n_actions; a.decisions = d_decisions; a.metrics = d_metrics;
    CK(vm_launch(e, a));
    return 0;
}
int maro_vm_step(MaroVmEnv* e, const uint8_t* active, const int32_t* actions, const int32_t* n_actions, int32_t* decisions,
                 int64_t* metrics) {
    if (!e || !decisions || !metrics) return fail("maro_vm_step: bad arguments");
    CK(cudaSetDevice(e->device));
    return common_host_step(e, active, actions, n_actions, decisions, metrics,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_vm_step_device(e, a, ac, na, d, m);
                            });
}
int maro_vm_pinned_buffers(MaroVmEnv* e, void** actions, void** n_actions, void** active, void** decisions, void** metrics) {
    return common_pinned_buffers(e, actions, n_actions, active, decisions, metrics);
}
int maro_vm_step_pinned(MaroVmEnv* e, int32_t use_actions, int32_t use_n_actions, int32_t use_active) {
    if (!e) return fail("maro_vm_step_pinned: null handle");
    CK(cudaSetDevice(e->device));
    const uint8_t* f = reinterpret_cast<const uint8_t*>(1);
    return common_host_step(e, use_active ? f : nullptr, use_actions ? reinterpret_cast<const int32_t*>(f) : nullptr,
                            use_n_actions ? reinterpret_cast<const int32_t*>(f) : nullptr, nullptr, nullptr,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_vm_step_device(e, a, ac, na, d, m);
                            }, true);
}
int maro_vm_query(MaroVmEnv* e, const int32_t* replicas, int32_t n_replicas, int32_t node_type, const int32_t* frame_indices,
                  int32_t n_frames, const int32_t* nodes, int32_t n_nodes, const int32_t* attrs, int32_t n_attrs, double* out,
                  int64_t* out_per_replica) {
    if (!out) return fail("maro_vm_query: null output");
    return query_impl(e, replicas, n_replicas, node_type, frame_indices, n_frames, nodes, n_nodes, attrs, n_attrs, nullptr, out, out_per_replica);
}
int maro_vm_save(MaroVmEnv* e, const char* path, int32_t with_snapshots) { return common_save(e, path, with_snapshots); }
int maro_vm_load(MaroVmEnv* e, const char* path) { return common_load(e, path); }
int maro_vm_set_query_layout(MaroVmEnv* e, int32_t layout) { return common_set_query_layout(e, layout); }
int32_t maro_vm_attr_id(MaroVmEnv* e, int32_t node_type, const char* name) { return common_attr_id(e, node_type, name); }
int32_t maro_vm_attr_slots(MaroVmEnv* e, int32_t node_type, int32_t attr_id) { return common_attr_slots(e, node_type, attr_id); }
int maro_vm_read_frame(MaroVmEnv* e, int32_t replica, int32_t* out_words, int32_t n_words) { return common_read_frame(e, replica, out_words, n_words); }
int maro_vm_ticks(MaroVmEnv* e, int32_t* out_ticks) { return common_ticks(e, out_ticks); }
int maro_vm_counters(MaroVmEnv* e, int64_t* out) { return common_counters(e, out); }
int maro_vm_snapshot_frames(MaroVmEnv* e, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out) {
    return common_snapshot_frames(e, replica, out, cap, n_out);
}
int maro_vm_rollout_device(MaroVmEnv* e, int32_t n_steps, int32_t* d_decisions, int64_t* d_metrics) {
    if (!e || !d_decisions || !d_metrics || n_steps < 1) return fail("maro_vm_rollout_device: bad arguments");
    CK(cudaSetDevice(e->device));
    VmArgs a = vm_base_args(e);
    a.decisions = d_decisions; a.metrics = d_metrics; a.n_steps = n_steps;
    const int w = e->warps_per_cta;
    const size_t smem = (size_t)w * vm_rollout_warp_bytes(e->s.N, e->s.DW);
    auto go = [&](auto kernel) -> cudaError_t {
        if (smem > 48 * 1024) {
            cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (err != cudaSuccess) return err;
        }
        kernel<<<e->grid, w * 32, smem, e->stream>>>(e->s, a);
        return cudaGetLastError();
    };
    CK(w == 1 ? go(vm_rollout_kernel<1>) : (w == 2 ? go(vm_rollout_kernel<2>) : go(vm_rollout_kernel<4>)));
    return 0;
}

int maro_vm_best_fit_policy_device(MaroVmEnv* e, const int32_t* d_decisions, int32_t* d_actions) {
    if (!e || !d_decisions || !d_actions) return fail("maro_vm_best_fit_policy_device: bad arguments");
    CK(cudaSetDevice(e->device));
    int threads = 128, blocks = std::min((e->B * 32 + threads - 1) / threads, e->n_sm * 16);
    vm_best_fit_kernel<<<blocks, threads, 0, e->stream>>>(e->s, e->d_state, d_decisions, d_actions);
    CK(cudaGetLastError());
    return 0;
}

}  // extern "C"

