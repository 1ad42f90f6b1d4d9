// cim_env.cu — kernels + C ABI (include/maro_b200.h) of the batched CIM discrete-event core for sm_90a (H100).
//
// Kernels
//   cim_step_kernel    one warp = one replica.  The replica's state block (frame | control | event queue) is
//                      staged HBM -> shared memory with one TMA bulk copy (cp.async.bulk + mbarrier), the step
//                      runs out of shared memory (cim_core.cuh), snapshot rows stream to the ring with 128-bit
//                      coalesced stores, and the block is written back with 128-bit stores.
//   cim_reset_kernel   Env.reset for masked replicas.
//   cim_query_kernel   snapshot_list[node][ticks:nodes:attrs] gather -> float64 (env_common.cuh, shared by the scenarios).
//   cim_policy_kernel  hashed random agent (bench helper).
//   cim_rl_*_kernel    RL state / action / reward shaping over the snapshot ring.
// The citi_bike and vm_scheduling scenarios are bike_env.cu / vm_env.cu (same handle layout, env_common.cuh).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
//   (-fmad=false: CPython never contracts a*b+c; order generation must round like the reference.)
#include "env_common.cuh"
#include <time.h>

#include <atomic>
#include <mutex>

// =====================================================================================================
// Kernels
// =====================================================================================================
struct StepArgs {
    int32_t* state;        // [B][SW]
    int32_t* snap;         // [B][ring][FWp]
    int32_t* snap_frame;   // [B][ring]
    uint32_t* mt;          // [B][MTW] or nullptr
    const int32_t* tables; // [K][table_words]
    const int32_t* replica_topology;  // [B]
    const uint8_t* active;            // [B] or nullptr
    const int32_t* actions;           // [B][A][4] or nullptr
    const int32_t* n_actions;         // [B] or nullptr
    int32_t* decisions;               // [B][8]
    int64_t* metrics;                 // [B][3]
    uint8_t* light;                   // [B] 1: the next step only applies an action and yields the tick's next decision
    int mt_words;
};

__device__ __forceinline__ Replica make_replica(const CimShape& s, const StepArgs& a, int rep, int32_t* st) {
    Replica r;
    r.f = st;
    r.c = st + s.FWp;
    r.q = st + s.FWp + s.CWp;
    r.t = a.tables + (int64_t)a.replica_topology[rep] * s.table_words;
    r.mt = a.mt ? a.mt + (int64_t)rep * a.mt_words : nullptr;
    r.snap = a.snap + (int64_t)rep * s.ring_rows * s.FWp;
    r.snap_frame = a.snap_frame + (int64_t)rep * s.ring_rows;
#ifdef MARO_PHASE_CLOCKS
    r.pc = nullptr;
#endif
    return r;
}

#ifdef MARO_PHASE_CLOCKS
__device__ unsigned long long maro_phase_clk[PH_SLOTS];  // summed over the replicas of every resident rollout
#endif

// kSpread (small batches, G < 32): one replica per WARP, only its first G lanes work.  Packing 32/G replicas into a warp
// makes the warp issue the union of their control paths; with fewer replicas than the GPU has warp slots it is faster to
// give every replica its own warp (same lane-group code, the other lanes exit).
template <int kWarps, int G, bool kGeneral, bool kSpread = false>
__global__ void __launch_bounds__(kWarps * 32, kGeneral ? 1 : 32 / kWarps) cim_step_kernel(const __grid_constant__ CimShape s,
                                                               const __grid_constant__ StepArgs a) {
    constexpr int kGroups = kSpread ? kWarps : kWarps * 32 / G;  // replicas in flight per CTA
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);  // one mbarrier per lane group (first 256 B)
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
    for (int rep = blockIdx.x * kGroups + gid; rep < s.n_replicas; rep += gridDim.x * kGroups) {
        if (a.active && !a.active[rep]) {
            if (g.lane == 0) a.decisions[(int64_t)rep * s.DW + 6] = MARO_STATUS_INACTIVE;
            continue;
        }
        int32_t* gstate = a.state + (int64_t)rep * s.SW;
        // ---- stage in: one TMA bulk copy, completion on the group's mbarrier.  A step that is known to stay inside
        // the current tick (another decision of the same tick is pending: it applies the action, snapshots and returns)
        // never touches the event queue, so only [frame | control] travels, both ways.
        const bool light = a.light[rep] != 0;
        const uint32_t bytes = light ? (uint32_t)(s.FWp + s.CWp) * 4u : (uint32_t)s.SW * 4u;
        if (g.lane == 0) {
            fence_proxy_async();  // order earlier generic-proxy accesses to this smem before the async write
            mbar_expect_tx(bar, bytes);
            bulk_g2s(st, gstate, bytes, bar);
        }
        while (!mbar_try_wait(bar, phase)) {}
        phase ^= 1u;
        Replica r = make_replica(s, a, rep, st);
        const int n_raw = a.actions ? (a.n_actions ? a.n_actions[rep] : 1) : 0;
        const bool too_many = n_raw > s.max_actions;  // more actions than the handle's rows hold: MARO_STATUS_BAD_ACTION
        const int n_act = too_many ? 1 : min(max(n_raw, 0), min(s.max_actions, G));
        Act4 act = {0, 0, 0, 0};
        if (g.lane < n_act) {  // lane k fetches action k with one 128-bit load (actions may live in mapped host memory)
            int4 v = reinterpret_cast<const int4*>(a.actions + (int64_t)rep * s.max_actions * 4)[g.lane];
            act.v = too_many ? -1 : v.x; act.p = v.y; act.qty = v.z; act.type = v.w;
        }
        replica_step<G, kGeneral>(s, g, r, act, n_act, a.decisions + (int64_t)rep * s.DW, a.metrics + (int64_t)rep * 3);
        // ---- write back (128-bit coalesced) what this step could have changed
        if (g.lane == 0) snapshot_drain_lane();
        const int4* src4 = reinterpret_cast<const int4*>(st);
        int4* dst4 = reinterpret_cast<int4*>(gstate);
        const int n4 = (int)(bytes >> 4);
        for (int i = g.lane; i < n4; i += G) dst4[i] = src4[i];
        if (g.lane == 0) {  // hint for the next step: awaiting an action with another arrival of this tick still to decide
            const int32_t* c = st + s.FWp;
            const uint64_t arr = ((uint64_t)(uint32_t)c[C_ARR_HI] << 32) | (uint32_t)c[C_ARR_LO];
            const int dp = c[C_DEC_POS];
            a.light[rep] = (c[C_STATE] == ST_AWAIT && dp < 64 && (arr >> dp) != 0) ? 1 : 0;
        }
        g.sync();
    }
}

__global__ void cim_reset_kernel(const __grid_constant__ CimShape s, const __grid_constant__ StepArgs a) {
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const Grp<32> g(threadIdx.x & 31);
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    for (int rep = warp_global; rep < s.n_replicas; rep += n_warps) {
        if (a.active && !a.active[rep]) continue;
        Replica r = make_replica(s, a, rep, a.state + (int64_t)rep * s.SW);  // operate directly on global memory
        replica_reset<32>(s, g, r);
        if (g.lane == 0) a.light[rep] = 0;
    }
}

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

// hello-world random agent (examples/hello_world/cim/hello.py:24-32) as a counter hash of (replica, step)
__device__ __forceinline__ int4 policy_random_row(const int32_t* d, uint32_t seed, uint32_t rid) {
    const uint32_t step = (uint32_t)d[7];
    uint32_t h1 = hash_u32(seed ^ hash_u32(rid * 0x9e3779b9u + step * 0x85ebca6bu + 0x1234567u));
    uint32_t h2 = hash_u32(h1 + 0x68bc21ebu);
    int load = d[3], dis = d[4];
    bool to_discharge = dis > 0 && (h1 & 1u);
    int scope = to_discharge ? dis : load;
    int qty = scope > 0 ? (int)(h2 % (uint32_t)(scope + 1)) : 0;
    return make_int4(d[2], d[1], qty, to_discharge ? 1 : 0);
}

__global__ void cim_policy_kernel(const int32_t* __restrict__ dec, int32_t* __restrict__ act, int n, int max_actions,
                                  uint32_t seed, uint32_t replica_base) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    *reinterpret_cast<int4*>(act + (int64_t)i * max_actions * 4) = policy_random_row(dec + i * 8, seed, (uint32_t)i + replica_base);
}

// =====================================================================================================
// Resident kernel: the replica block stays in shared memory for MANY env-steps (DESIGN.md §5 "resident mode").
//   mode RES_ROLLOUT  K fused env-steps per launch, the agent is a device callback evaluated between the steps
//                     (null / hashed hello-world agent); per step only the snapshot rows (and an optional 32-byte
//                     trace row) leave the SM.  No co-residency requirement: any batch size.
//   mode RES_SESSION  host-driven: the kernel stays resident between Env.step calls; per step the host writes one
//                     16-byte command row per replica {seq, flags, vessel|port<<16, qty} into mapped pinned memory,
//                     the replica's lane group polls it over PCIe, steps, writes its decision + metrics rows to mapped
//                     pinned memory and bumps a device counter; the last group publishes `seq` to a host flag.
//                     Groups that see no command for `idle_cycles` write back and exit (the host relaunches).
// Stage-in (one TMA bulk copy) and write-back happen once per launch instead of once per env-step.
// =====================================================================================================
enum { RES_ROLLOUT = 0, RES_SESSION = 1 };
enum { RES_POLICY_NULL = 0, RES_POLICY_RANDOM = 1 };
enum { RES_CMD_STEP = 0, RES_CMD_EXIT = 1 };
// result line of the session: MARO_RES_LINE_CHUNKS tagged 16-byte chunks (see "publish" in the session loop)
#define MARO_RES_LINE_CHUNKS 5
#define MARO_RES_LINE_WORDS (4 * MARO_RES_LINE_CHUNKS)
// command row word 1 (flags): bits 0-7 n_actions | bit 8 active | bit 9 bad action | bit 10 Env.reset before the step |
//                             bits 16-23 command | bit 24 action type of row 0
struct ResidentArgs {
    int mode, spread;
    int n_steps, policy;
    uint32_t seed, replica_base;
    int32_t* trace;                 // [n_steps][B][8] decision rows of every fused step, or nullptr
    int slice_steps;                // RES_ROLLOUT, sliced: > 0 = lane groups pull (replica, slice of `slice_steps` env-steps) work items
    uint32_t* slice_sync;           //   device: {tickets taken, entries appended, entries[B x (n_slices - 1)]}, zeroed before the launch
    const uint32_t* cmd;            // [B][4] command rows (mapped host memory)
    uint32_t* results;              // mapped host [B][MARO_RES_LINE_WORDS]: tagged result lines (see "publish" in the session loop)
    uint32_t poll_ns, wait_ns;      // back-off of the command poll (PCIe) and of the shared-memory relay wait
    uint32_t* seq_state;            // device [B]: last seq each replica has completed (survives launches and resets)
    int32_t* rows;                  // device [B][16]: each replica's decision + metrics slot between launches of the session
    const uint32_t* heartbeat;      // mapped host word the host bumps while it is inside submit / wait (any thread)
    uint32_t* exit_flag;            // device word: set (to `epoch`) by the first CTA that gives up waiting; every CTA of the launch
    uint32_t epoch;                 //   leaves at its next poll once it is set, so a launch never ends for only SOME of its CTAs
    long long idle_cycles;
};

__device__ __forceinline__ uint4 ld_sys_v4(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

// kMinBlocks = 3 caps the kernel's registers (no spills either way).  It helps grids several waves deep and costs at smaller
// ones (toy.4p, fused rollouts) -- so it is chosen per handle (res_dense) once the grid is several waves deep.  Shared memory, not registers, bounds residency here (2 CTAs per SM in both builds).
#ifndef MARO_RES_DENSE_BLOCKS
#define MARO_RES_DENSE_BLOCKS 3
#endif
// kSmall: the small-topology instantiation of replica_step (cim_small_ok), chosen per handle at create (res_small).
template <int G, bool kGeneral, int kMinBlocks = 1, bool kSmall = false>
__global__ void __launch_bounds__(256, kMinBlocks) cim_resident_kernel(const __grid_constant__ CimShape s, const __grid_constant__ StepArgs a,
                                                           const __grid_constant__ ResidentArgs ra) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int n_groups = ra.spread ? (int)(blockDim.x >> 5) : (int)(blockDim.x / G);
    if (ra.spread && (threadIdx.x & 31) >= G) return;
    const int gid = ra.spread ? (int)(threadIdx.x >> 5) : (int)(threadIdx.x / G);
    int rep = blockIdx.x * n_groups + gid;
    const Grp<G> g(threadIdx.x & 31);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw) + gid;                  // [32] mbarriers
    int32_t* dslot = reinterpret_cast<int32_t*>(smem_raw + 256) + gid * 16;      // 8 decision words + 3 int64 metrics
    int64_t* mslot = reinterpret_cast<int64_t*>(dslot + 8);
    int32_t* st = reinterpret_cast<int32_t*>(smem_raw + 256 + (size_t)n_groups * 64) + (size_t)gid * s.SW;
    // Sliced rollouts (grids that do not fit the GPU at once, e.g. 1.16 waves): instead of one replica per lane group for the whole
    // launch, the resident lane groups serve a FIFO of ready replicas.  A work item is one slice = `slice_steps` env-steps of one
    // replica between a stage-in and a write-back; the group that finishes a slice appends the replica (with its next slice number)
    // to the queue — release / acquire on the queue entry hands the block over through global memory, possibly to another SM.
    // Entries are written once (the queue has B x (n_slices - 1) of them, tickets < B are the replicas' first slices), a group only
    // ever waits for an entry that a running slice will write: no deadlock, no wait while any replica is ready.  The makespan
    // becomes work / resident groups instead of ceil(waves) x the rollout time.
    const bool sliced = ra.mode == RES_ROLLOUT && ra.slice_steps > 0;
    const int n_slices = sliced ? (ra.n_steps + ra.slice_steps - 1) / ra.slice_steps : 1;
    int k_begin = 0, k_end = ra.n_steps, slice = 0;
    uint32_t phase = 0;
    if (g.lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
    }
    if (!sliced && rep >= s.n_replicas) return;
  for (;;) {
    if (sliced) {
        uint32_t v = 0;
        if (g.lane == 0) {
            const uint32_t B = (uint32_t)s.n_replicas;
            const uint32_t t = atomicAdd(ra.slice_sync, 1u);
            if (t >= B * (uint32_t)n_slices) v = 0xffffffffu;
            else if (t < B) v = t + 1u;
            else
                for (;;) {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ra.slice_sync + 2 + (t - B)) : "memory");
                    if (v) break;
                    __nanosleep(100);
                }
        }
        v = (uint32_t)g.shfl((int)v, 0);
        if (v == 0xffffffffu) return;
        slice = (int)(v >> 24);
        rep = (int)(v & 0xffffffu) - 1;
        k_begin = slice * ra.slice_steps;
        k_end = min(ra.n_steps, k_begin + ra.slice_steps);
    }
    int32_t* gstate = a.state + (int64_t)rep * s.SW;
    if (g.lane == 0) {
        if (sliced) asm volatile("fence.proxy.async;" ::: "memory");  // (the block in global memory was written by generic stores of another group)
        fence_proxy_async();
        mbar_expect_tx(bar, (uint32_t)s.SW * 4u);
        bulk_g2s(st, gstate, (uint32_t)s.SW * 4u, bar);
    }
    g.sync();
    while (!mbar_try_wait(bar, phase)) {}
    phase ^= 1u;
    Replica r = make_replica(s, a, rep, st);
    Ctl k;  // the control state stays in registers until the write-back below
    ctl_load<G, kSmall>(s, g, r, k);
    int32_t* gdec = a.decisions + (int64_t)rep * 8;
    int64_t* gmet = a.metrics + (int64_t)rep * 3;

    if (ra.mode == RES_ROLLOUT) {
        if (g.lane < 8) dslot[g.lane] = gdec[g.lane];  // the decision the previous launch / slice returned (feeds the agent)
        if (slice > 0 && g.lane < 3) mslot[g.lane] = gmet[g.lane];
        g.sync();
        int step = k_begin;
        // (a later slice of a replica whose episode ended in an earlier one: nothing left to do but the trace rows)
        const bool over = slice > 0 && (dslot[MARO_DEC_STATUS] == MARO_STATUS_FINISHED || dslot[MARO_DEC_STATUS] == MARO_STATUS_DONE);
#ifdef MARO_PHASE_CLOCKS
        PhaseClk pclk;
        for (int i = 0; i < PH_SLOTS; i++) pclk.acc[i] = 0;
        pclk.t = clock64();
        r.pc = &pclk;
#endif
        for (; step < k_end && !over; step++) {
            PHASE_MARK(r, PH_STORE);  // (the previous step's trace row and status test)
            Act4 act = {0, 0, 0, 0};
            int n_act = 0;
            if (ra.policy == RES_POLICY_RANDOM) {
                n_act = 1;
                if (g.lane == 0) {
                    int4 o = policy_random_row(dslot, ra.seed, (uint32_t)rep + ra.replica_base);
                    act.v = o.x; act.p = o.y; act.qty = o.z; act.type = o.w;
                }
            }
            PHASE_MARK(r, PH_AGENT);
            PHASE_COUNT(r, PH_STEPS, 1);
            replica_step<G, kGeneral, kSmall, true>(s, g, r, k, act, n_act, dslot, mslot);
            if (ra.trace && g.lane < 2)
                reinterpret_cast<int4*>(ra.trace + ((int64_t)step * s.n_replicas + rep) * 8)[g.lane] = reinterpret_cast<const int4*>(dslot)[g.lane];
            const int status = dslot[MARO_DEC_STATUS];
            // the episode is over: stop here and keep the DONE row with the final metrics (a further step — in this launch
            // or the next — returns the all-zero FINISHED row, core.py:128-131)
            if (status == MARO_STATUS_FINISHED || status == MARO_STATUS_DONE) { step++; break; }
        }
#ifdef MARO_PHASE_CLOCKS
        PHASE_MARK(r, PH_STORE);
        if (g.lane == 0)
            for (int i = 0; i < PH_SLOTS; i++) atomicAdd(&maro_phase_clk[i], pclk.acc[i]);
        r.pc = nullptr;
#endif
        flush_deferred_snapshot<G, kSmall>(s, g, r, k);  // (the work item ends: its last decision's snapshot becomes observable)
        if (ra.trace)
            for (; step < k_end; step++)
                if (g.lane < 2)
                    reinterpret_cast<int4*>(ra.trace + ((int64_t)step * s.n_replicas + rep) * 8)[g.lane] = reinterpret_cast<const int4*>(dslot)[g.lane];
        if (g.lane < 2) reinterpret_cast<int4*>(gdec)[g.lane] = reinterpret_cast<const int4*>(dslot)[g.lane];
        if (g.lane < 3) gmet[g.lane] = mslot[g.lane];
    } else {
        // ---- host session.  Per CTA: group 0 polls the CTA's command rows (one coalesced PCIe read for all of them) and
        // relays them through shared memory; every group steps its replica into its output slot; the group that finishes
        // last copies all slots to the mapped host rows (coalesced), fences once and bumps the completion counter.
        uint32_t* cmd_s = reinterpret_cast<uint32_t*>(smem_raw + 256 + (size_t)n_groups * 64 + (size_t)n_groups * s.SW * 4);  // [n_groups][4]
        volatile uint32_t* seq_s = cmd_s + n_groups * 4;
        const int rep0 = blockIdx.x * n_groups;
        const int n_live = min(n_groups, s.n_replicas - rep0);
        uint32_t expect = ra.seq_state[rep0] + 1u;
        if (threadIdx.x == 0) *seq_s = expect - 1u;
        __syncthreads();  // (threads that left above do not take part in CTA barriers)
        // rows of inactive replicas keep their previous contents.  The slot outlives the launch in device memory: when the
        // kernel comes back up after an idle exit, the host may not have unpacked every result line of the last step yet.
        for (int i = g.lane; i < 16; i += G) dslot[i] = ra.rows[(int64_t)rep * 16 + i];
        g.sync();
        for (;;) {
            if (gid == 0) {
                long long t0 = clock64();
                uint32_t beat = 0;
                bool stop = false, have_beat = false;
                for (;;) {
                    bool ok = true;
                    // (issued ahead of the PCIe reads so that both are in flight together: has another CTA given up on this launch?)
                    uint32_t f = 0;
                    if (g.lane == 0) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(f) : "l"(ra.exit_flag) : "memory");
                    for (int b0 = 0; b0 < n_live; b0 += G) {
                        const int i = b0 + g.lane;
                        uint4 c = make_uint4(expect, 0, 0, 0);
                        if (i < n_live) c = ld_sys_v4(ra.cmd + (int64_t)(rep0 + i) * 4);
                        ok = ok && g.ballot(c.x != expect) == 0;
                        if (i < n_live) *reinterpret_cast<uint4*>(cmd_s + i * 4) = c;
                    }
                    if (ok) break;
                    // another CTA has given up: leave with it (the host relaunches the whole grid; a command that arrives
                    // meanwhile stays in its row and is picked up by the next launch) — a launch never ends for only SOME CTAs
                    if ((uint32_t)g.shfl((int)f, 0) == ra.epoch) { stop = true; break; }
                    if (g.shfl((int)(clock64() - t0 > ra.idle_cycles), 0)) {  // (the leader's clock decides for the group)
                        // no command for a while: leave only if the host has left submit / wait altogether (its heartbeat stands
                        // still) — then every CTA leaves within one idle period and the host relaunches the whole grid.  While
                        // any host thread is still driving other CTAs, a slow driver of this CTA must not strand it.
                        uint32_t b = 0;
                        if (g.lane == 0) asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(b) : "l"(ra.heartbeat) : "memory");
                        b = (uint32_t)g.shfl((int)b, 0);
                        if (have_beat && b == beat) {
                            if (g.lane == 0) atomicExch(ra.exit_flag, ra.epoch);
                            stop = true;
                            break;
                        }
                        beat = b; have_beat = true;
                        t0 = clock64();
                    }
                    if (ra.poll_ns) __nanosleep(ra.poll_ns);
                }
                if (stop)  // idle: every group of the CTA leaves together
                    for (int i = g.lane; i < n_live; i += G) cmd_s[i * 4 + 1] = (uint32_t)RES_CMD_EXIT << 16;
                g.sync();
                __threadfence_block();
                if (g.lane == 0) *seq_s = expect;
            }
            if (g.lane == 0) while (*seq_s != expect) if (ra.wait_ns) __nanosleep(ra.wait_ns);
            g.sync();
            __threadfence_block();
            const uint4 c = *reinterpret_cast<const uint4*>(cmd_s + gid * 4);
            const uint32_t flags = c.y;
            if (((flags >> 16) & 0xff) == RES_CMD_EXIT) break;
            const int n_act = min((int)(flags & 0xff), min(s.max_actions, G));
            const bool active = (flags >> 8) & 1u, bad = (flags >> 9) & 1u;
            if ((flags >> 10) & 1u) {  // Env.reset of this replica (maro_cim_reset while the session is live), in place
                ctl_store<G, kSmall>(s, g, r, k);  // (the work counters in registers survive the reset)
                replica_reset<G>(s, g, r);
                ctl_load<G, kSmall>(s, g, r, k);
            }
            if (active) {
                Act4 act = {0, 0, 0, 0};
                if (g.lane == 0) {
                    act.v = bad ? -1 : (int)(c.z & 0xffffu); act.p = (int)(c.z >> 16); act.qty = (int)c.w; act.type = (int)((flags >> 24) & 1u);
                } else if (g.lane < n_act) {  // further actions of an action list: full rows in the pinned action buffer
                    __threadfence_system();  // (acquire side of the host's release store of the command row)
                    uint4 v = ld_sys_v4(reinterpret_cast<const uint32_t*>(a.actions + ((int64_t)rep * s.max_actions + g.lane) * 4));
                    act.v = (int)v.x; act.p = (int)v.y; act.qty = (int)v.z; act.type = (int)v.w;
                }
                replica_step<G, kGeneral, kSmall>(s, g, r, k, act, n_act, dslot, mslot);
            } else if (g.lane == 0) {
                dslot[MARO_DEC_STATUS] = MARO_STATUS_INACTIVE;
            }
            g.sync();
            // ---- publish: one 80-byte result line per replica in mapped host memory, five 16-byte chunks, each written by ONE
            // 128-bit store that carries the sequence number in its last word.  The 14 payload words (decision words 0..7, then
            // the metrics as 3 x int64 — dslot and mslot are contiguous) go three to a chunk:
            //     chunk c = payload words 3c, 3c+1, 3c+2 | seq          (word 14 of the payload is padding)
            // The host takes a line once all five tags show the step it is waiting for — no system fence, no separate flag
            // (a 16-byte aligned store reaches host memory as one write: tag and payload become visible together).
            if (g.lane < MARO_RES_LINE_CHUNKS) {
                const uint32_t* p = reinterpret_cast<const uint32_t*>(dslot);
                uint32_t w[3];
#pragma unroll
                for (int i = 0; i < 3; i++) {
                    const int wi = 3 * g.lane + i;
                    w[i] = wi < 14 ? p[wi] : 0u;
                }
                asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(ra.results + (int64_t)rep * MARO_RES_LINE_WORDS + g.lane * 4),
                             "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(expect)
                             : "memory");
            }
            expect++;
        }
        if (g.lane == 0) ra.seq_state[rep] = expect - 1u;
        for (int i = g.lane; i < 16; i += G) ra.rows[(int64_t)rep * 16 + i] = dslot[i];
    }
    // ---- write back the block + the light-step hint of the per-step kernel
    ctl_store<G, kSmall>(s, g, r, k);
    if (g.lane == 0) snapshot_drain_lane();
    g.sync();
    const int4* src4 = reinterpret_cast<const int4*>(st);
    int4* dst4 = reinterpret_cast<int4*>(gstate);
    for (int i = g.lane; i < s.SW / 4; i += G) dst4[i] = src4[i];
    if (g.lane == 0) {
        const int32_t* c = st + s.FWp;
        const uint64_t arr = ((uint64_t)(uint32_t)c[C_ARR_HI] << 32) | (uint32_t)c[C_ARR_LO];
        const int dp = c[C_DEC_POS];
        a.light[rep] = (c[C_STATE] == ST_AWAIT && dp < 64 && (arr >> dp) != 0) ? 1 : 0;
    }
    if (!sliced) return;
    __threadfence();  // (every lane: its part of the block, the decision / metrics rows and the snapshot rows it drained)
    g.sync();
    if (g.lane == 0 && slice + 1 < n_slices) {
        const uint32_t at = atomicAdd(ra.slice_sync + 1, 1u);
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(ra.slice_sync + 2 + at), "r"(((uint32_t)(slice + 1) << 24) | (uint32_t)(rep + 1)) : "memory");
    }
  }
}

enum { kMaxSlices = 16 };
struct ResGeom { int threads = 0, grid = 0; size_t smem = 0; int per_sm = 0; };  // launch shape of cim_resident_kernel

struct MaroCimEnv : EnvCommon {
    CimShape s;
    int K = 0, mt_words = 0, warps_per_cta = 4, lanes = 32, grid = 0, max_stops = 0, max_targets = 0, max_distinct = 0;
    bool spread = false;  // one replica per warp (cim_step_kernel kSpread)
    size_t smem_bytes = 0;
    int32_t *d_tables = nullptr, *d_topo = nullptr;
    uint32_t* d_mt = nullptr;
    uint8_t* d_light = nullptr;
    std::vector<int32_t> h_tables;
    // resident mode (cim_resident_kernel)
    int res_threads = 0, res_grid = 0, res_spread = 0, res_dense = 0;
    int res_small = 0;                               // the resident kernel runs the small-topology instantiation (cim_small_ok)
    size_t res_smem = 0;
    bool session_ok = false;                         // the whole grid is co-resident (required to spin-wait)
    std::atomic<bool> session_live{false};
    std::mutex session_mu;                           // launch / relaunch / end of the resident kernel (submit / wait of DISJOINT
                                                     // CTA ranges may run on several host threads at once)
    std::vector<uint8_t> reset_pending;              // per replica: maro_cim_reset arrived while the session was live -> rides on
                                                     // the replica's next command row (or is applied when the session ends)
    uint32_t *h_beat = nullptr, *hd_beat = nullptr;  // heartbeat word, mapped pinned
    uint32_t* d_slice = nullptr;                     // sliced rollouts: ready queue, 2 + B x (kMaxSlices - 1) words
    int res_per_sm = 0, res_slice_steps = -1;        // resident CTAs per SM; steps per slice (-1 = decide per launch, 0 = never)
    uint32_t* d_exit = nullptr;                      // exit flag of the resident kernel (device), compared with launch_epoch
    uint32_t launch_epoch = 0;
    int buf_full_cap = 1, buf_empty_cap = 1;         // buffer ticks the event pool was sized for (set_topology re-validation)
    int res_groups = 0;                              // replicas per CTA of the resident kernel
    ResGeom roll;                                    // launch shape of the fused rollouts
    std::vector<uint32_t> cta_seq;                   // per CTA: last step completed (the kernel's seq_state mirrors it)
    std::vector<uint8_t> cta_pending;                // per CTA: a step has been sent and not collected yet
    uint32_t *h_cmd = nullptr, *hd_cmd = nullptr;    // [B][4] command rows, mapped pinned
    uint32_t *h_res = nullptr, *hd_res = nullptr;    // [B][MARO_RES_LINE_WORDS] tagged result lines, mapped pinned (16-byte aligned chunks)
    uint32_t* d_seq = nullptr;
    int32_t* d_rows = nullptr;                       // [B][16] decision + metrics slots of the session (ResidentArgs::rows)
    long long idle_cycles = 400000;
    uint32_t poll_ns = 0, wait_ns = 20;
};

// =====================================================================================================
// RL state / reward shaping on the snapshot ring (SURVEY.md §8f rank 1; examples/cim/rl/env_sampler.py:15-36, 66-80)
// =====================================================================================================
struct ShapeArgs {
    const int32_t* snap;
    const int32_t* snap_frame;
    int ring_rows, FWp, B;
    // state
    const int32_t* decisions;  // [B][8]
    int look_back_ticks;       // look_back - 1 frames: max(0, tick - rt), rt = 0..look_back-2
    int n_ports_per_state;     // 1 + future_stop_number
    int npa, nva;              // attribute counts
    int port_attr_off[16], port_attr_isf[16], vessel_attr_off[16], vessel_attr_isf[16];
    int o_fut, fut;            // future_stop_list: word offset, slots per vessel
    int P, V;
    double* state_out;         // [B][look_back_ticks * n_ports_per_state * npa + nva]
    float* state_out_f32;      // the same rounded to float32 (what the example feeds its networks), when state_out is null
    // reward
    const int32_t* ticks;      // [B] tick of the action
    const int32_t* ports;      // [B] port that acted
    const double* decay;       // [time_window] time_decay ** i
    int time_window, off_fulfillment, off_shortage;
    int n_rows;                // rewards for [n_rows][B] (tick, port) pairs in one launch (row-major; replica = item % B)
    double fulfillment_factor, shortage_factor;
    float* reward_out;         // [B]
    // action translation
    const int32_t* model_actions;  // [B] index into action_space
    const double* action_space;    // [n_action_space]
    int n_action_space, finite_vessel_space, has_early_discharge, max_actions, off_remaining_space, off_early_discharge;
    int32_t* actions_out;          // [B][max_actions][4]
    // sampler extras of the action kernel (maro_cim_rl_action_ex_device), each optional
    const int64_t* model_actions_i64;  // [B] the policy's output as int64 (torch argmax) instead of model_actions
    int32_t* model_actions_record;     // [B] the index that was used, as int32 (the sampler's record)
    const int64_t* met_in;             // [B][3] metrics of the previous step ...
    int64_t* met_final;                // [B][3] ... folded into a running maximum (= the metrics of the DONE row, see rl_rollout.py)
};

// word `w` of snapshot `frame` of replica `rep`; frames not in the ring read as 0 (np_backend.pyx:543-549)
__device__ __forceinline__ bool snap_row(const ShapeArgs& q, int rep, int frame, const int32_t*& row) {
    if (frame < 0) return false;
    int r = frame % q.ring_rows;
    if (q.snap_frame[(int64_t)rep * q.ring_rows + r] != frame) return false;
    row = q.snap + ((int64_t)rep * q.ring_rows + r) * q.FWp;
    return true;
}

// state[rep] = concat(ports[ticks : [port] + future_stop_list : port_attrs], vessels[tick : vessel : vessel_attrs]) as float64
__global__ void cim_rl_state_kernel(const __grid_constant__ ShapeArgs q) {
    const int per_tick = q.n_ports_per_state * q.npa;
    const int dim = q.look_back_ticks * per_tick + q.nva;
    const int64_t total = (int64_t)q.B * dim;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int rep = (int)(i / dim), e = (int)(i % dim);
        const int32_t* d = q.decisions + (int64_t)rep * 8;
        double v = 0.0;
        if (d[MARO_DEC_STATUS] == MARO_STATUS_DECISION) {
            const int tick = d[MARO_DEC_TICK], vessel = d[MARO_DEC_VESSEL];
            const int32_t* now = nullptr;
            const bool have_now = snap_row(q, rep, tick, now);
            if (e >= q.look_back_ticks * per_tick) {
                const int a = e - q.look_back_ticks * per_tick;
                if (have_now) {
                    int w = now[q.vessel_attr_off[a] + vessel];
                    v = q.vessel_attr_isf[a] ? (double)__int_as_float(w) : (double)w;
                }
            } else {
                const int k = e / per_tick, j = (e % per_tick) / q.npa, a = e % q.npa;
                int port = d[MARO_DEC_PORT];
                if (j > 0) port = have_now ? now[q.o_fut + vessel * q.fut + (j - 1)] : 0;  // .astype("int") of a 0-padded query
                const int frame = tick - k > 0 ? tick - k : 0;
                const int32_t* row = nullptr;
                if (port >= 0 && port < q.P && snap_row(q, rep, frame, row)) {
                    int w = row[q.port_attr_off[a] + port];
                    v = q.port_attr_isf[a] ? (double)__int_as_float(w) : (double)w;
                }
            }
        }
        if (q.state_out) q.state_out[i] = v;
        else q.state_out_f32[i] = (float)v;
    }
}

// reward[rep] = float32(ff * sum_k decay[k] * fulfillment[tick+1+k, port] - sf * sum_k decay[k] * shortage[tick+1+k, port])
__global__ void cim_rl_reward_kernel(const __grid_constant__ ShapeArgs q) {
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int n_warps = (gridDim.x * blockDim.x) >> 5;
    const int64_t n_items = (int64_t)q.n_rows * q.B;
    for (int64_t item = warp_global; item < n_items; item += n_warps) {
        const int rep = (int)(item % q.B);
        const int tick = q.ticks[item], port = q.ports[item];
        double f = 0.0, sh = 0.0;
        if (port >= 0 && port < q.P && tick >= 0) {
            for (int k = lane; k < q.time_window; k += 32) {
                const int32_t* row = nullptr;
                if (snap_row(q, rep, tick + 1 + k, row)) {
                    f += q.decay[k] * (double)row[q.off_fulfillment + port];
                    sh += q.decay[k] * (double)row[q.off_shortage + port];
                }
            }
        }
        for (int o = 16; o > 0; o >>= 1) {
            f += __shfl_xor_sync(0xffffffffu, f, o);
            sh += __shfl_xor_sync(0xffffffffu, sh, o);
        }
        if (lane == 0) q.reward_out[item] = (float)(q.fulfillment_factor * f - q.shortage_factor * sh);
    }
}

static void register_attrs(MaroCimEnv* e) {
    const CimShape& s = e->s;
    static const char* pn[] = {"acc_booking", "acc_fulfillment", "acc_shortage", "booking", "capacity", "empty",
                               "fulfillment", "full", "on_consignee", "on_shipper", "shortage", "transfer_cost"};
    for (int a = 0; a < 12; a++) e->attrs[0].push_back({pn[a], a * s.P, 1, a == 11, s.P});
    static const char* vn[] = {"capacity", "early_discharge", "empty", "full", "is_parking", "last_loc_idx",
                               "loc_port_idx", "next_loc_idx", "remaining_space", "route_idx"};
    for (int a = 0; a < 10; a++) e->attrs[1].push_back({vn[a], s.o_vs + a * s.V, 1, 0, s.V});
    e->attrs[1].push_back({"past_stop_list", s.o_past, s.past, 0, s.V});
    e->attrs[1].push_back({"past_stop_tick_list", s.o_past_tick, s.past, 0, s.V});
    e->attrs[1].push_back({"future_stop_list", s.o_fut, s.fut, 0, s.V});
    e->attrs[1].push_back({"future_stop_tick_list", s.o_fut_tick, s.fut, 0, s.V});
    e->attrs[2].push_back({"full_on_ports", s.o_fop, s.P * s.P, 0, 1});
    e->attrs[2].push_back({"full_on_vessels", s.o_fov, s.V * s.P, 0, 1});
    e->attrs[2].push_back({"vessel_plans", s.o_vp, s.V * s.P, 0, 1});
}

static StepArgs base_args(MaroCimEnv* e) {
    StepArgs a;
    memset(&a, 0, sizeof(a));
    a.state = e->d_state;
    a.snap = e->d_snap;
    a.snap_frame = e->d_snap_frame;
    a.mt = e->d_mt;
    a.tables = e->d_tables;
    a.replica_topology = e->d_topo;
    a.light = e->d_light;
    a.mt_words = e->mt_words;
    return a;
}

template <int W, int G, bool kGeneral>
static cudaError_t launch_step_wgn(MaroCimEnv* e, const StepArgs& a) {
    if (G < 32 && W == 4 && e->spread) {  // one replica per warp (small batches), instantiated for 4 warps per CTA only
        cudaError_t err = cudaFuncSetAttribute(cim_step_kernel<W, G, kGeneral, (G < 32 && W == 4)>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem_bytes);
        if (err != cudaSuccess) return err;
        cim_step_kernel<W, G, kGeneral, (G < 32 && W == 4)><<<e->grid, W * 32, e->smem_bytes, e->stream>>>(e->s, a);
        return cudaGetLastError();
    }
    cudaError_t err = cudaFuncSetAttribute(cim_step_kernel<W, G, kGeneral>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem_bytes);
    if (err != cudaSuccess) return err;
    cim_step_kernel<W, G, kGeneral><<<e->grid, W * 32, e->smem_bytes, e->stream>>>(e->s, a);
    return cudaGetLastError();
}

template <int W, int G>
static cudaError_t launch_step_wg(MaroCimEnv* e, const StepArgs& a) {
    // noise-free fixed-mode topologies run the specialised kernel (no MT19937 / float64 paths compiled in)
    const bool general = !(e->s.order_table && !e->s.buffer_noise);
    return general ? launch_step_wgn<W, G, true>(e, a) : launch_step_wgn<W, G, false>(e, a);
}

template <int G>
static cudaError_t launch_step_g(MaroCimEnv* e, const StepArgs& a) {
    switch (e->warps_per_cta) {
        case 1: return launch_step_wg<1, G>(e, a);
        case 2: return launch_step_wg<2, G>(e, a);
        case 4: return launch_step_wg<4, G>(e, a);
        default: return launch_step_wg<8, G>(e, a);
    }
}

static cudaError_t launch_step(MaroCimEnv* e, const StepArgs& a) {
    switch (e->lanes) {
        case 8: return launch_step_g<8>(e, a);
        case 16: return launch_step_g<16>(e, a);
        default: return launch_step_g<32>(e, a);
    }
}

template <int G>
static cudaError_t launch_resident_g(MaroCimEnv* e, const StepArgs& a, const ResidentArgs& ra, const ResGeom& geo, bool query_only,
                                     int* blocks_per_sm) {
    const bool general = !(e->s.order_table && !e->s.buffer_noise);
    auto go = [&](auto kernel) -> cudaError_t {
        cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)geo.smem);
        if (err != cudaSuccess) return err;
        if (query_only) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, kernel, geo.threads, geo.smem);
        kernel<<<geo.grid, geo.threads, geo.smem, e->stream>>>(e->s, a, ra);
        return cudaGetLastError();
    };
    if (general) return go(cim_resident_kernel<G, true>);
    if (e->res_small) return go(cim_resident_kernel<G, false, 1, true>);
    return e->res_dense ? go(cim_resident_kernel<G, false, MARO_RES_DENSE_BLOCKS>) : go(cim_resident_kernel<G, false>);
}

static cudaError_t launch_resident(MaroCimEnv* e, const StepArgs& a, const ResidentArgs& ra, const ResGeom& geo, bool query_only = false,
                                   int* blocks_per_sm = nullptr) {
    switch (e->lanes) {
        case 8: return launch_resident_g<8>(e, a, ra, geo, query_only, blocks_per_sm);
        case 16: return launch_resident_g<16>(e, a, ra, geo, query_only, blocks_per_sm);
        default: return launch_resident_g<32>(e, a, ra, geo, query_only, blocks_per_sm);
    }
}
static ResGeom session_geom(const MaroCimEnv* e) { return ResGeom{e->res_threads, e->res_grid, e->res_smem, e->res_per_sm}; }

// ---- host session (RES_SESSION) ---------------------------------------------------------------------
// Threading contract: maro_cim_submit_pinned / maro_cim_wait_pinned may be called concurrently from several host threads as
// long as their replica ranges are disjoint (per-CTA bookkeeping is touched by the owning thread only; launching, relaunching
// and ending the kernel are serialised by session_mu).  Every other entry point is single-threaded, like the rest of the ABI.
static inline void session_beat(MaroCimEnv* e) { __atomic_fetch_add(e->h_beat, 1u, __ATOMIC_RELAXED); }

static int session_launch_locked(MaroCimEnv* e) {
    StepArgs a = base_args(e);
    a.actions = reinterpret_cast<const int32_t*>(e->hd_in);
    a.decisions = reinterpret_cast<int32_t*>(e->hd_out);
    a.metrics = reinterpret_cast<int64_t*>(e->hd_out + (size_t)e->B * e->dec_words * 4);
    ResidentArgs ra;
    memset(&ra, 0, sizeof(ra));
    ra.mode = RES_SESSION; ra.spread = e->res_spread;
    ra.cmd = e->hd_cmd; ra.results = e->hd_res; ra.seq_state = e->d_seq; ra.rows = e->d_rows; ra.poll_ns = e->poll_ns; ra.wait_ns = e->wait_ns;
    ra.idle_cycles = e->idle_cycles; ra.heartbeat = e->hd_beat;
    ra.exit_flag = e->d_exit; ra.epoch = ++e->launch_epoch;  // (epochs start at 1; the flag holds 0 or an older epoch)
    CK(launch_resident(e, a, ra, session_geom(e)));
    e->session_live.store(true, std::memory_order_release);
    return 0;
}

// Wait until the CTAs [c0, c1) have published the step they were last sent (their decision / metrics rows are then in
// h_out).  The resident kernel may have left meanwhile (the host was away for longer than the idle limit): relaunch it,
// the command rows are still in place.
static int session_wait_ctas(MaroCimEnv* e, int c0, int c1) {
    const int gpc = e->res_groups, B = e->B;
    int32_t* dec = reinterpret_cast<int32_t*>(e->h_out);
    int64_t* met = reinterpret_cast<int64_t*>(e->h_out + (size_t)B * e->dec_words * 4);
    timespec ts0;
    clock_gettime(CLOCK_MONOTONIC, &ts0);
    int cta = c0, rep = c0 * gpc;
    // take the result lines in order; a line is complete when every chunk tag carries the awaited sequence number
    auto advance = [&]() {
        while (cta < c1) {
            if (!e->cta_pending[cta]) { cta++; rep = cta * gpc; continue; }
            const uint32_t want = e->cta_seq[cta] + 1u;
            const int end = std::min(B, (cta + 1) * gpc);
            while (rep < end) {
                const volatile uint32_t* line = e->h_res + (size_t)rep * MARO_RES_LINE_WORDS;
                for (int c = 0; c < MARO_RES_LINE_CHUNKS; c++)
                    if (line[4 * c + 3] != want) return false;
                __atomic_thread_fence(__ATOMIC_ACQUIRE);  // (x86: loads are not reordered; this stops the compiler)
                const uint32_t* l = const_cast<const uint32_t*>(line);
                uint32_t p[3 * MARO_RES_LINE_CHUNKS];  // payload: decision words 0..7, metrics 3 x int64
                for (int c = 0; c < MARO_RES_LINE_CHUNKS; c++) memcpy(p + 3 * c, l + 4 * c, 12);
                memcpy(dec + (size_t)rep * 8, p, 32);
                memcpy(met + (size_t)rep * 3, p + 8, 24);
                rep++;
            }
            e->cta_pending[cta] = 0;
            e->cta_seq[cta] += 1u;
            cta++;
        }
        return true;
    };
    for (uint64_t spins = 1;; spins++) {
        if (advance()) return 0;
        __builtin_ia32_pause();
        if ((spins & 0x3ff) == 0) session_beat(e);  // (every ~25 us: "the host is still here", see the kernel's idle exit)
        if ((spins & 0xfff) == 0) {  // every ~100 us: did the kernel leave (idle limit) or fail?
            timespec ts;
            clock_gettime(CLOCK_MONOTONIC, &ts);
            if (ts.tv_sec - ts0.tv_sec > 30) return fail("resident kernel: no completion after 30 s");  // never spin forever
            if (cudaStreamQuery(e->stream) == cudaErrorNotReady) continue;
            std::lock_guard<std::mutex> lock(e->session_mu);
            cudaError_t q = cudaStreamQuery(e->stream);  // (another waiting thread may have relaunched it already)
            if (q == cudaSuccess) {
                if (advance()) return 0;
                if (session_launch_locked(e)) return 1;
            } else if (q != cudaErrorNotReady) {
                e->session_live.store(false);
                return fail(std::string("resident kernel: ") + cudaGetErrorString(q));
            }
        }
    }
}

extern "C" int maro_cim_reset(MaroCimEnv* e, const uint8_t* mask);
static int reset_now(MaroCimEnv* e, const uint8_t* mask);

// Ask the resident kernel (if any) to write the replica blocks back and exit; afterwards device memory is authoritative.
static int session_end(MaroCimEnv* e) {
    if (!e->session_live.load()) return 0;
    bool any = false;
    for (int c = 0; c < e->res_grid; c++) any = any || e->cta_pending[c];
    if (any && session_wait_ctas(e, 0, e->res_grid)) return 1;
    {
        std::lock_guard<std::mutex> lock(e->session_mu);
        const int gpc = e->res_groups;
        for (int i = 0; i < e->B; i++) {
            volatile uint32_t* row = e->h_cmd + (size_t)i * 4;
            row[1] = (uint32_t)RES_CMD_EXIT << 16;
            __atomic_store_n(&row[0], e->cta_seq[i / gpc] + 1u, __ATOMIC_RELEASE);
        }
        e->session_live.store(false);
        CK(cudaStreamSynchronize(e->stream));
        // the EXIT rows must not be taken for commands by the next launch (a CTA whose first command row has not been written
        // yet when the kernel comes up would leave at once): park every row on a sequence number nobody waits for
        for (int i = 0; i < e->B; i++) __atomic_store_n(e->h_cmd + (size_t)i * 4, e->cta_seq[i / gpc], __ATOMIC_RELEASE);
    }
    // resets that arrived while the session was live and never rode on a command row
    bool pend = false;
    for (int i = 0; i < e->B; i++) pend = pend || e->reset_pending[i];
    if (pend) {
        std::vector<uint8_t> m(e->reset_pending);
        std::fill(e->reset_pending.begin(), e->reset_pending.end(), (uint8_t)0);
        if (reset_now(e, m.data())) return 1;
    }
    return 0;
}
#define END_SESSION(e) do { if ((e)->session_live.load() && session_end(e)) return 1; } while (0)

// Send one Env.step to the replicas [first, first + count) (whole CTAs): one 16-byte command row per replica, built from
// the pinned staging buffers (h_in).  Returns at once; session_wait_ctas collects the rows.
static int session_submit(MaroCimEnv* e, int first, int count, bool use_actions, bool use_n_actions, bool use_active) {
    const int B = e->B, A = e->s.max_actions, gpc = e->res_groups;
    if (first < 0 || count < 1 || first + count > B || first % gpc || ((first + count) % gpc && first + count != B))
        return fail("submit: the replica range must cover whole blocks of maro_cim_pinned_granularity() replicas");
    const int c0 = first / gpc, c1 = (first + count + gpc - 1) / gpc;
    for (int c = c0; c < c1; c++)
        if (e->cta_pending[c]) { if (session_wait_ctas(e, c0, c1)) return 1; break; }
    const int32_t* act = reinterpret_cast<const int32_t*>(e->h_in);
    const int32_t* nact = reinterpret_cast<const int32_t*>(e->h_in + (size_t)B * A * 16);
    const uint8_t* active = e->h_in + (size_t)B * A * 16 + (size_t)B * 4;
    for (int i = first; i < first + count; i++) {
        int n = use_actions ? (use_n_actions ? nact[i] : 1) : 0;
        if (n < 0) n = 0;
        const int32_t* r0 = act + (size_t)i * A * 4;
        const bool is_active = use_active ? active[i] != 0 : true;
        uint32_t flags = (is_active ? 1u : 0u) << 8, w2 = 0, w3 = 0;
        if (e->reset_pending[i]) {  // (a replica outside the active mask is still reset: Env.reset does not depend on stepping)
            flags |= 1u << 10;
            e->reset_pending[i] = 0;
        }
        if (n > 0) {
            const bool bad = n > A || r0[0] < 0 || r0[0] > 0xffff || r0[1] < 0 || r0[1] > 0xffff;
            flags |= (uint32_t)std::min(n, 255) | (bad ? 1u << 9 : 0u) | (r0[3] == 1 ? 1u << 24 : 0u);
            w2 = ((uint32_t)r0[0] & 0xffffu) | ((uint32_t)r0[1] << 16);
            w3 = (uint32_t)r0[2];
        }
        volatile uint32_t* row = e->h_cmd + (size_t)i * 4;
        row[1] = flags; row[2] = w2; row[3] = w3;
        __atomic_store_n(&row[0], e->cta_seq[i / gpc] + 1u, __ATOMIC_RELEASE);  // x86 TSO: a reader that sees the seq sees the row
    }
    __atomic_thread_fence(__ATOMIC_SEQ_CST);
    for (int c = c0; c < c1; c++) e->cta_pending[c] = 1;
    session_beat(e);
    if (!e->session_live.load(std::memory_order_acquire)) {
        std::lock_guard<std::mutex> lock(e->session_mu);
        if (!e->session_live.load() && session_launch_locked(e)) return 1;
    }
    return 0;
}

// One Env.step of every replica through the resident kernel (inputs in h_in, outputs in h_out, both mapped).
static int session_step(MaroCimEnv* e, bool use_actions, bool use_n_actions, bool use_active) {
    if (session_submit(e, 0, e->B, use_actions, use_n_actions, use_active)) return 1;
    return session_wait_ctas(e, 0, e->res_grid);
}

// device buffers + resident-mode geometry of a new handle; any failure leaves the handle for the caller to destroy
static int create_device_side(MaroCimEnv* e, const MaroCimTopology* topos, int32_t n_topos, const MaroCimConfig* cfg, const cudaDeviceProp& prop) {
    (void)topos;
    const CimShape& s = e->s;
    const int B = e->B;
    CK(cudaMalloc(&e->d_tables, e->h_tables.size() * 4));
    CK(cudaMalloc(&e->d_topo, (size_t)B * 4));
    CK(cudaMalloc(&e->d_light, (size_t)B));
    CK(cudaMemset(e->d_light, 0, (size_t)B));
    CK(cudaMemcpy(e->d_tables, e->h_tables.data(), e->h_tables.size() * 4, cudaMemcpyHostToDevice));
    std::vector<int32_t> topo(B, 0);
    if (cfg->replica_topology)
        for (int i = 0; i < B; i++) {
            if (cfg->replica_topology[i] < 0 || cfg->replica_topology[i] >= n_topos) return fail("maro_cim_create: replica_topology out of range");
            topo[i] = cfg->replica_topology[i];
        }
    CK(cudaMemcpy(e->d_topo, topo.data(), (size_t)B * 4, cudaMemcpyHostToDevice));
    if (s.order_noise || s.buffer_noise) {
        e->mt_words = mt_block_words(s);
        CK(cudaMalloc(&e->d_mt, (size_t)B * e->mt_words * 4));
    }
    // ---- resident mode: one replica per warp while the batch is small (spread), packed lane groups otherwise
    CK(cudaHostAlloc(&e->h_cmd, (size_t)B * 16, cudaHostAllocMapped));
    CK(cudaHostAlloc(&e->h_res, (size_t)B * MARO_RES_LINE_WORDS * 4, cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer((void**)&e->hd_cmd, e->h_cmd, 0));
    CK(cudaHostGetDevicePointer((void**)&e->hd_res, e->h_res, 0));
    memset(e->h_cmd, 0, (size_t)B * 16);
    memset(e->h_res, 0, (size_t)B * MARO_RES_LINE_WORDS * 4);
    CK(cudaMalloc(&e->d_seq, (size_t)B * 4));
    CK(cudaMemset(e->d_seq, 0, (size_t)B * 4));
    CK(cudaMalloc(&e->d_rows, (size_t)B * 64));
    CK(cudaMemset(e->d_rows, 0, (size_t)B * 64));  // (= the zeroed host rows the first session starts from)
    CK(cudaMalloc(&e->d_slice, (2 + (size_t)B * (kMaxSlices - 1)) * 4));
    CK(cudaMalloc(&e->d_exit, 64));
    CK(cudaMemset(e->d_exit, 0, 64));
    CK(cudaHostAlloc(&e->h_beat, 64, cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer((void**)&e->hd_beat, e->h_beat, 0));
    memset(e->h_beat, 0, 64);
    e->reset_pending.assign(B, 0);
    const int nsm = prop.multiProcessorCount;
    const int gpw = 32 / e->lanes;
    const size_t per_group = (size_t)s.SW * 4 + 64 + 16, max_smem = prop.sharedMemPerBlockOptin;  // block + output slot + command row
    // One replica per warp (spread) while every replica can be resident at once, else 32 / lanes replicas per warp (packed).  The
    // resident kernel holds fewer warps per SM than the per-step kernel: a spread grid that needs more than one wave is slower than
    // the packed one, one that fits is faster.  MARO_B200_RES_SPREAD=0/1 forces a mode.
    const char* rs = getenv("MARO_B200_RES_SPREAD");
    e->res_spread = rs ? atoi(rs) != 0 : (B <= nsm * 32);
    e->n_sm = nsm;
    for (int attempt = 0; attempt < 2; attempt++) {
        const int groups_per_warp = e->res_spread ? 1 : gpw;
        int w = 8;
        if (e->res_spread) {  // smallest power of two >= replicas per SM (command blocks of a CTA stay 64 / 128-byte aligned)
            w = 1;
            while (w < 8 && w * nsm < B) w <<= 1;
        }
        if (const char* rw = getenv("MARO_B200_RES_WARPS")) w = std::min(8, std::max(1, atoi(rw)));
        while (w > 1 && 256 + 16 + per_group * w * groups_per_warp > max_smem) w--;
        e->res_threads = 0;
        if (256 + 16 + per_group * w * groups_per_warp > max_smem) break;  // (the block does not fit: per-step kernel only)
        e->res_threads = w * 32;
        e->res_smem = 256 + 16 + per_group * w * groups_per_warp;
        e->res_grid = (B + w * groups_per_warp - 1) / (w * groups_per_warp);
        e->res_groups = w * groups_per_warp;
        const char* rd = getenv("MARO_B200_RES_DENSE");  // register-capped instantiation for grids several waves deep
        e->res_dense = rd ? atoi(rd) != 0 : (!e->res_spread && w == 8 && e->res_grid > 5 * nsm);
        int per_sm = 0;
        StepArgs a = base_args(e);
        ResidentArgs ra;
        memset(&ra, 0, sizeof(ra));
        e->res_small = 0;
        CK(launch_resident(e, a, ra, session_geom(e), true, &per_sm));
        // the small-topology instantiation where the shape allows it (MARO_B200_RES_SMALL=0/1 forces it off / on where allowed),
        // never in place of the register-capped one and never where it would hold fewer CTAs per SM
        const char* rsm = getenv("MARO_B200_RES_SMALL");
        if (cim_small_ok(s, e->lanes) && (rsm ? atoi(rsm) != 0 : !e->res_dense)) {
            int per_sm_small = 0;
            e->res_small = 1;
            CK(launch_resident(e, a, ra, session_geom(e), true, &per_sm_small));
            if (per_sm_small < per_sm && !rsm) e->res_small = 0;
            else per_sm = per_sm_small;
        }
        e->res_per_sm = per_sm;
        if (attempt == 0 && e->res_spread && !rs && gpw > 1 && (int64_t)per_sm * nsm < e->res_grid) {
            e->res_spread = 0;
            continue;
        }
        // Rollouts use the session's launch shape.  (The CTA size is not a lever: the kernel is latency bound per warp, not
        // balance bound per SM.  MARO_B200_ROLL_WARPS forces a CTA size for A/B runs.)
        e->roll = session_geom(e);
        if (const char* fw = getenv("MARO_B200_ROLL_WARPS")) {
            const int cw = std::min(w, std::max(1, atoi(fw)));
            ResGeom g;
            g.threads = cw * 32;
            g.smem = 256 + 16 + per_group * cw * groups_per_warp;
            g.grid = (B + cw * groups_per_warp - 1) / (cw * groups_per_warp);
            CK(launch_resident(e, a, ra, g, true, &g.per_sm));
            e->roll = g;
        }
        e->cta_seq.assign(e->res_grid, 0);
        e->cta_pending.assign(e->res_grid, 0);
        if (const char* sl = getenv("MARO_B200_RES_SLICE_STEPS")) e->res_slice_steps = atoi(sl);
        const char* se = getenv("MARO_B200_SESSION");
        e->session_ok = (se ? atoi(se) != 0 : true) && (int64_t)per_sm * nsm >= e->res_grid && !s.joint;  // (fixed-size result lines)
        break;
    }
    e->scenario_id = 1;
    e->ckpt_extra = {{"tables", (void**)&e->d_tables, e->h_tables.size() * 4}, {"replica_topology", (void**)&e->d_topo, (size_t)B * 4},
                     {"mt19937", (void**)&e->d_mt, (size_t)B * e->mt_words * 4}, {"light", (void**)&e->d_light, (size_t)B}};
    if (const char* v = getenv("MARO_B200_POLL_NS")) e->poll_ns = (uint32_t)atoi(v);
    if (const char* v = getenv("MARO_B200_WAIT_NS")) e->wait_ns = (uint32_t)atoi(v);
    if (const char* iu = getenv("MARO_B200_IDLE_US")) e->idle_cycles = (long long)(atof(iu) * 1e-6 * prop.clockRate * 1e3);
    return maro_cim_reset(e, nullptr);
}

extern "C" {

const char* maro_last_error(void) {
    if (g_err.empty()) {  // nothing failed on this thread: the latest failure of any thread (worker threads of a host loop)
        std::lock_guard<std::mutex> lock(g_err_mu);
        g_err = g_err_any;
    }
    return g_err.c_str();
}
int maro_abi_version(void) { return MARO_B200_ABI_VERSION; }

int maro_cim_destroy(MaroCimEnv* e) {
    if (!e) return 0;
    cudaSetDevice(e->device);
    if (e->session_live.load()) session_end(e);
    cudaFree(e->d_tables); cudaFree(e->d_topo); cudaFree(e->d_mt); cudaFree(e->d_light);
    cudaFree(e->d_seq); cudaFree(e->d_rows); cudaFree(e->d_exit); cudaFree(e->d_slice);
    if (e->h_cmd) cudaFreeHost(e->h_cmd);
    if (e->h_res) cudaFreeHost(e->h_res);
    if (e->h_beat) cudaFreeHost(e->h_beat);
    common_free(e);
    delete e;
    return 0;
}

int maro_cim_create(const MaroCimTopology* topos, int32_t n_topos, const MaroCimConfig* cfg, MaroCimEnv** out) {
    if (!topos || n_topos < 1 || !cfg || !out || cfg->n_replicas < 1) return fail("maro_cim_create: bad arguments");
    const MaroCimTopology& t0 = topos[0];
    if (t0.n_ports < 1 || t0.n_ports > 255 || t0.n_vessels < 1 || t0.n_vessels > 64)
        return fail("maro_cim_create: supported sizes are 1..255 ports and 1..64 vessels");
    for (int k = 1; k < n_topos; k++)
        if (check_same_shape(t0, topos[k])) return fail("maro_cim_create: all topologies of one handle must share a shape");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail("maro_cim_create: no CUDA device — this library has no CPU path");
    if (cfg->device < 0 || cfg->device >= ndev) return fail("maro_cim_create: bad device ordinal");
    CK(cudaSetDevice(cfg->device));

    MaroCimEnv* e = new MaroCimEnv();
    e->device = cfg->device;
    e->B = cfg->n_replicas;
    e->K = n_topos;
    CimShape& s = e->s;
    if (compute_shape_and_tables(topos, n_topos, cfg, s, e->h_tables, e->max_stops, e->max_targets, e->max_distinct)) {
        delete e;
        return fail("maro_cim_create: inconsistent topology tables / durations must be positive");
    }
    for (int k = 0; k < n_topos; k++) {
        const CimTopoNeeds n = topology_needs(topos[k]);
        e->buf_full_cap = std::max(e->buf_full_cap, n.buf_full);
        e->buf_empty_cap = std::max(e->buf_empty_cap, n.buf_empty);
    }
    if (cfg->queue_capacity > 0) e->buf_full_cap = e->buf_empty_cap = 1 << 30;  // explicit pool size: the caller's responsibility
    const char* ln = getenv("MARO_B200_LANES");  // tuning override: lanes per replica (8 / 16 / 32, >= the topology's minimum)
    const int cfg_lanes = ln ? std::max(atoi(ln), lanes_per_replica(s)) : 0;
    register_attrs(e);

    // launch geometry: G lanes per replica, as many warps per CTA as shared memory allows (<= 8), persistent grid
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, e->device) != cudaSuccess) { delete e; return fail("maro_cim_create: cudaGetDeviceProperties failed"); }
    e->lanes = cfg_lanes > 0 ? cfg_lanes : lanes_per_replica(s);
    const int gpw = 32 / e->lanes;  // replicas per warp
    const size_t per_warp = (size_t)s.SW * 4 * gpw;
    const size_t max_smem = prop.sharedMemPerBlockOptin;
    if (256 + per_warp > max_smem) { delete e; return fail("maro_cim_create: replica state does not fit in shared memory"); }
    // warps per CTA: the choice that keeps the most warps resident per SM (shared memory vs the 64-register budget
    // of the specialised kernel), then fewer for small batches so that replicas spread over all SMs
    const size_t sm_smem = prop.sharedMemPerMultiprocessor;
    int w = 1, best = 0;
    for (int cand = 8; cand >= 1; cand >>= 1) {
        size_t cta = 256 + per_warp * cand;
        if (cta > max_smem) continue;
        int blocks = (int)std::min<size_t>(sm_smem / (cta + 1024), (size_t)(64 / cand));
        if (blocks * cand > best) { best = blocks * cand; w = cand; }
    }
    while (w > 1 && (e->B + w * gpw - 1) / (w * gpw) < prop.multiProcessorCount) w >>= 1;
    e->warps_per_cta = w;
    e->smem_bytes = 256 + per_warp * w;
    int ctas_needed = (e->B + w * gpw - 1) / (w * gpw);
    int resident = std::max<int>(1, (int)std::min<size_t>(64 / w, sm_smem / (e->smem_bytes + 1024)));
    e->grid = std::min(ctas_needed, prop.multiProcessorCount * resident);
    // small batch, sub-warp groups: one replica per warp while the replicas fit the resident warp slots (<= 32 per SM)
    const char* sp = getenv("MARO_B200_SPREAD");
    const bool want_spread = sp ? atoi(sp) != 0 : e->B <= prop.multiProcessorCount * 32;  // every replica gets a resident warp
    if (gpw > 1 && want_spread && 256 + (size_t)s.SW * 4 * 4 <= max_smem) {
        e->spread = true;
        e->warps_per_cta = 4;
        e->smem_bytes = 256 + (size_t)s.SW * 4 * 4;
        e->grid = (e->B + 3) / 4;
    }

    e->ring_rows = s.ring_rows; e->FW = s.FW; e->FWp = s.FWp; e->SW = s.SW;
    e->off_tick = s.FWp + C_TICK; e->off_counters = s.FWp + C_NSTEPS_LO;
    e->dec_words = s.DW; e->max_actions = s.max_actions;
    if (common_alloc(e)) { maro_cim_destroy(e); return 1; }
    int rc = create_device_side(e, topos, n_topos, cfg, prop);
    if (rc) { maro_cim_destroy(e); return rc; }
    *out = e;
    return 0;
}

int maro_cim_set_stream(MaroCimEnv* e, void* cuda_stream, int32_t external) {
    if (!e) return fail("null handle");
    END_SESSION(e);
    e->stream = external ? (cudaStream_t)cuda_stream : e->own_stream;
    return 0;
}

int maro_cim_reset(MaroCimEnv* e, const uint8_t* mask) {
    if (!e) return fail("null handle");
    CK(cudaSetDevice(e->device));
    if (e->session_live.load()) {
        // The replica blocks live in shared memory right now: the reset rides on each replica's next command row and is
        // carried out there, in place (replica_reset in the resident kernel) — no write-back / relaunch round trip.  Calls that
        // read device state end the session first, which applies whatever is still pending (session_end).
        bool busy = false;
        const int gpc = e->res_groups;
        for (int i = 0; i < e->B; i++)
            if ((!mask || mask[i]) && e->cta_pending[i / gpc]) busy = true;
        if (!busy) {
            for (int i = 0; i < e->B; i++)
                if (!mask || mask[i]) e->reset_pending[i] = 1;
            return 0;
        }
        if (session_end(e)) return 1;  // a step of these replicas is still in flight: the conservative path
    }
    return reset_now(e, mask);
}
}  // extern "C"

static int reset_now(MaroCimEnv* e, const uint8_t* mask) {
    StepArgs a = base_args(e);
    if (mask) {
        if (common_stage_mask(e, mask, &a.active)) return 1;
        for (int i = 0; i < e->B; i++) if (mask[i]) e->reset_pending[i] = 0;
    } else {
        std::fill(e->reset_pending.begin(), e->reset_pending.end(), (uint8_t)0);
    }
    int threads = 128, blocks = std::min((e->B * 32 + threads - 1) / threads, e->n_sm * 16);
    cim_reset_kernel<<<blocks, threads, 0, e->stream>>>(e->s, a);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

extern "C" {

int maro_cim_set_topology(MaroCimEnv* e, int32_t index, const MaroCimTopology* topo) {
    if (!e || !topo || index < 0 || index >= e->K) return fail("maro_cim_set_topology: bad arguments");
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    std::vector<int32_t> blob;
    if (topo->n_ports != e->s.P || topo->n_vessels != e->s.V || topo->max_tick != e->s.max_tick)
        return fail("maro_cim_set_topology: shape differs from the handle's");
    if (topo->stop_offset[topo->n_vessels] > e->max_stops || topo->target_offset[topo->n_ports] > e->max_targets)
        return fail("maro_cim_set_topology: more stops/targets than the handle was sized for");
    {   // the handle's calendar-queue horizon, default queue capacity and RNG paths were sized from the create-time
        // topologies: a replacement has to fit them (an event beyond the horizon would alias into an earlier bucket)
        const CimTopoNeeds n = topology_needs(*topo);
        if (e->s.due_R && !n.stops_increase)  // (the due-ring drain takes one stop per vessel and tick)
            return fail("maro_cim_set_topology: the new instance has a vessel whose stop ticks do not strictly increase; the handle "
                        "keeps its discharges per stop (create the handle with this instance among its topologies)");
        if (!e->s.due_R && n.max_delay + 1 > e->s.QH)
            return fail("maro_cim_set_topology: the new instance needs an event horizon of " + std::to_string(n.max_delay + 1) +
                        " ticks, the handle was created with " + std::to_string(e->s.QH) + " (create the handle with this instance among its topologies)");
        if ((n.order_noise && !e->s.order_noise) || (n.buffer_noise && !e->s.buffer_noise))
            return fail("maro_cim_set_topology: the new instance draws order / buffer noise, the handle was created without those streams");
        if (n.buf_full > e->buf_full_cap || n.buf_empty > e->buf_empty_cap)
            return fail("maro_cim_set_topology: longer container buffer times than the handle's event pool was sized for");
    }
    CimShape probe = e->s;  // rebuild with identical padding; offsets must come out the same
    if ((e->s.order_table && count_distinct_orders(*topo) > e->max_distinct) ||
        build_blob(*topo, probe, blob, e->max_stops, e->max_targets, true, e->max_distinct) || probe.table_words != e->s.table_words ||
        probe.t_mt_buffer != e->s.t_mt_buffer || probe.t_order_proportion != e->s.t_order_proportion)
        return fail("maro_cim_set_topology: shape differs from the handle's");
    memcpy(e->h_tables.data() + (size_t)index * e->s.table_words, blob.data(), blob.size() * 4);
    CK(cudaMemcpy(e->d_tables + (size_t)index * e->s.table_words, blob.data(), blob.size() * 4, cudaMemcpyHostToDevice));
    return 0;
}

int maro_cim_step_device(MaroCimEnv* e, const uint8_t* d_active, const int32_t* d_actions, const int32_t* d_n_actions,
                         int32_t* d_decisions, int64_t* d_metrics) {
    if (!e || !d_decisions || !d_metrics) return fail("maro_cim_step_device: bad arguments");
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    StepArgs a = base_args(e);
    a.active = d_active; a.actions = d_actions; a.n_actions = d_n_actions;
    a.decisions = d_decisions; a.metrics = d_metrics;
    CK(launch_step(e, a));
    return 0;
}

int maro_cim_step(MaroCimEnv* e, const uint8_t* active, const int32_t* actions, const int32_t* n_actions,
                  int32_t* decisions, int64_t* metrics) {
    if (!e || !decisions || !metrics) return fail("maro_cim_step: bad arguments");
    CK(cudaSetDevice(e->device));
    if (e->session_ok) {  // resident kernel: stage through the pinned buffers, command rows out, decision rows back
        const int B = e->B, A = e->s.max_actions;
        const size_t act_bytes = (size_t)B * A * 16, dec_bytes = (size_t)B * e->dec_words * 4;
        if (actions) memcpy(e->h_in, actions, act_bytes);
        if (actions && n_actions) memcpy(e->h_in + act_bytes, n_actions, (size_t)B * 4);
        if (active) memcpy(e->h_in + act_bytes + (size_t)B * 4, active, B);
        if (session_step(e, actions != nullptr, actions && n_actions, active != nullptr)) return 1;
        memcpy(decisions, e->h_out, dec_bytes);
        memcpy(metrics, e->h_out + dec_bytes, (size_t)B * e->met_words * 8);
        return 0;
    }
    return common_host_step(e, active, actions, n_actions, decisions, metrics,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_cim_step_device(e, a, ac, na, d, m);
                            });
}

int maro_cim_pinned_buffers(MaroCimEnv* e, void** actions, void** n_actions, void** active, void** decisions, void** metrics) {
    return common_pinned_buffers(e, actions, n_actions, active, decisions, metrics);
}
int maro_cim_step_pinned(MaroCimEnv* e, int32_t use_actions, int32_t use_n_actions, int32_t use_active) {
    if (!e) return fail("maro_cim_step_pinned: null handle");
    CK(cudaSetDevice(e->device));
    if (e->session_ok) return session_step(e, use_actions != 0, use_actions && use_n_actions, use_active != 0);
    const uint8_t* f = reinterpret_cast<const uint8_t*>(1);  // presence flags only
    return common_host_step(e, use_active ? f : nullptr, use_actions ? reinterpret_cast<const int32_t*>(f) : nullptr,
                            use_n_actions ? reinterpret_cast<const int32_t*>(f) : nullptr, nullptr, nullptr,
                            [&](const uint8_t* a, const int32_t* ac, const int32_t* na, int32_t* d, int64_t* m) {
                                return maro_cim_step_device(e, a, ac, na, d, m);
                            }, true);
}
int32_t maro_cim_pinned_granularity(MaroCimEnv* e) { return e && e->session_ok ? e->res_groups : 0; }
int maro_cim_submit_pinned(MaroCimEnv* e, int32_t first, int32_t count, int32_t use_actions, int32_t use_n_actions, int32_t use_active) {
    if (!e) return fail("maro_cim_submit_pinned: null handle");
    if (!e->session_ok) return fail("maro_cim_submit_pinned: the batch is not resident (maro_cim_pinned_granularity() == 0); use maro_cim_step_pinned");
    CK(cudaSetDevice(e->device));
    return session_submit(e, first, count, use_actions != 0, use_actions && use_n_actions, use_active != 0);
}
int maro_cim_wait_pinned(MaroCimEnv* e, int32_t first, int32_t count) {
    if (!e || !e->session_ok || first < 0 || count < 1 || first + count > e->B) return fail("maro_cim_wait_pinned: bad arguments");
    CK(cudaSetDevice(e->device));
    return session_wait_ctas(e, first / e->res_groups, (first + count + e->res_groups - 1) / e->res_groups);
}
int32_t maro_cim_frame_words(MaroCimEnv* e) { return e ? e->s.FW : -1; }

int maro_cim_query(MaroCimEnv* e, const int32_t* replicas, int32_t n_replicas, int32_t node_type, const int32_t* frame_indices,
                   int32_t n_frames, const int32_t* nodes, int32_t n_nodes, const int32_t* attrs, int32_t n_attrs, double* out,
                   int64_t* out_per_replica) {
    if (!out) return fail("maro_cim_query: null output");
    if (e) END_SESSION(e);
    return query_impl(e, replicas, n_replicas, node_type, frame_indices, n_frames, nodes, n_nodes, attrs, n_attrs, nullptr, out, out_per_replica);
}

int maro_cim_query_device(MaroCimEnv* e, const int32_t* replicas, int32_t n_replicas, int32_t node_type, const int32_t* frame_indices,
                          int32_t n_frames, const int32_t* nodes, int32_t n_nodes, const int32_t* attrs, int32_t n_attrs, double* d_out,
                          int64_t* out_per_replica) {
    if (!d_out) return fail("maro_cim_query_device: null output");
    if (e) END_SESSION(e);
    return query_impl(e, replicas, n_replicas, node_type, frame_indices, n_frames, nodes, n_nodes, attrs, n_attrs, d_out, nullptr, out_per_replica);
}

/* Env.dump / restore: the whole simulation state of the handle (replica blocks, snapshot ring, RNG streams, topology tables) */
int maro_cim_save(MaroCimEnv* e, const char* path, int32_t with_snapshots) {
    if (e) END_SESSION(e);
    return common_save(e, path, with_snapshots);
}
int maro_cim_load(MaroCimEnv* e, const char* path) {
    if (e) END_SESSION(e);
    int rc = common_load(e, path);
    if (!rc) {  // host mirror of the topology tables (set_topology edits it in place)
        CK(cudaMemcpy(e->h_tables.data(), e->d_tables, e->h_tables.size() * 4, cudaMemcpyDeviceToHost));
        std::fill(e->reset_pending.begin(), e->reset_pending.end(), (uint8_t)0);
    }
    return rc;
}
int maro_cim_set_query_layout(MaroCimEnv* e, int32_t layout) { return common_set_query_layout(e, layout); }
int32_t maro_cim_attr_id(MaroCimEnv* e, int32_t node_type, const char* name) { return common_attr_id(e, node_type, name); }
int32_t maro_cim_attr_slots(MaroCimEnv* e, int32_t node_type, int32_t attr_id) { return common_attr_slots(e, node_type, attr_id); }
int maro_cim_read_frame(MaroCimEnv* e, int32_t replica, int32_t* out_words, int32_t n_words) {
    if (e) END_SESSION(e);
    return common_read_frame(e, replica, out_words, n_words);
}
int maro_cim_ticks(MaroCimEnv* e, int32_t* out_ticks) {
    if (e) END_SESSION(e);
    return common_ticks(e, out_ticks);
}
int maro_cim_counters(MaroCimEnv* e, int64_t* out) {
    if (e) END_SESSION(e);
    return common_counters(e, out);
}
int maro_cim_snapshot_frames(MaroCimEnv* e, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out) {
    if (e) END_SESSION(e);
    return common_snapshot_frames(e, replica, out, cap, n_out);
}

/* K fused env-steps per replica in ONE launch, the agent evaluated on the device between the steps. */
int maro_cim_rollout_device(MaroCimEnv* e, int32_t policy, uint32_t seed, uint32_t replica_base, int32_t n_steps,
                            int32_t* d_decisions, int64_t* d_metrics, int32_t* d_trace) {
    if (!e || !d_decisions || !d_metrics || n_steps < 1 || (policy != RES_POLICY_NULL && policy != RES_POLICY_RANDOM))
        return fail("maro_cim_rollout_device: bad arguments");
    if (!e->res_threads) return fail("maro_cim_rollout_device: replica state does not fit the resident kernel");
    if (e->s.joint) return fail("maro_cim_rollout_device: the device agents answer one decision at a time (Sequential mode)");
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    StepArgs a = base_args(e);
    a.decisions = d_decisions; a.metrics = d_metrics;
    ResidentArgs ra;
    memset(&ra, 0, sizeof(ra));
    ra.mode = RES_ROLLOUT; ra.spread = e->res_spread; ra.n_steps = n_steps; ra.policy = policy; ra.seed = seed;
    ra.replica_base = replica_base; ra.trace = d_trace;
    // Sliced launch when the grid does not fit the GPU at once and the last wave would be mostly empty (>= 10 % of the launch
    // lost to it): resident lane groups pull (slice, replica) tickets instead (cim_resident_kernel).
    ResGeom geo = e->roll;
    const int capacity = geo.per_sm * e->n_sm;
    int slice_steps = 0;
    // (one replica per warp only: lane groups that share a warp would serialise once they run different slices)
    const bool warp_per_replica = e->res_spread || e->lanes == 32;
    if (e->res_slice_steps > 0) slice_steps = e->res_slice_steps;  // (forced: tests, A/B)
    else if (e->res_slice_steps < 0 && capacity > 0 && geo.grid > capacity && n_steps >= 16) {
        const int waves = (geo.grid + capacity - 1) / capacity;
        if ((int64_t)waves * capacity * 10 >= (int64_t)geo.grid * 11) slice_steps = 8;
    }
    if (!warp_per_replica) slice_steps = 0;
    if (slice_steps) slice_steps = std::max(slice_steps, (n_steps + kMaxSlices - 1) / kMaxSlices);
    if (slice_steps >= n_steps || e->B >= (1 << 24) - 1) slice_steps = 0;
    if (slice_steps) {
        const int n_slices = (n_steps + slice_steps - 1) / slice_steps;
        CK(cudaMemsetAsync(e->d_slice, 0, (2 + (size_t)e->B * (n_slices - 1)) * 4, e->stream));
        ra.slice_steps = slice_steps; ra.slice_sync = e->d_slice;
        geo.grid = std::min(geo.grid, std::max(1, capacity));
    }
    CK(launch_resident(e, a, ra, geo));
    return 0;
}

#ifdef MARO_PHASE_CLOCKS
// (-DMARO_PHASE_CLOCKS builds only, tools/phase_clocks.py) copy the phase accumulators of the device to `out` [PH_SLOTS],
// then zero them if `clear`.  Synchronises the device.
int maro_cim_phase_clocks(uint64_t* out, int32_t clear) {
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyFromSymbol(out, maro_phase_clk, sizeof(unsigned long long) * PH_SLOTS));
    if (clear) {
        static const unsigned long long zero[PH_SLOTS] = {};
        CK(cudaMemcpyToSymbol(maro_phase_clk, zero, sizeof(zero)));
    }
    return 0;
}
#endif

int maro_cim_random_policy_device(MaroCimEnv* e, const int32_t* d_decisions, int32_t* d_actions, uint32_t seed,
                                  uint32_t replica_base) {
    if (!e || !d_decisions || !d_actions) return fail("maro_cim_random_policy_device: bad arguments");
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    int threads = 256, blocks = (e->B + threads - 1) / threads;
    cim_policy_kernel<<<blocks, threads, 0, e->stream>>>(d_decisions, d_actions, e->B, e->s.max_actions, seed, replica_base);
    CK(cudaGetLastError());
    return 0;
}

}  // extern "C"

// _translate_to_env_action (examples/cim/rl/env_sampler.py:38-64): model action index -> {vessel, port, quantity, type}
__global__ void cim_rl_action_kernel(const __grid_constant__ ShapeArgs q) {
    const int rep = blockIdx.x * blockDim.x + threadIdx.x;
    if (rep >= q.B) return;
    const int32_t* d = q.decisions + (int64_t)rep * 8;
    if (q.model_actions_record) q.model_actions_record[rep] = q.model_actions_i64 ? (int)q.model_actions_i64[rep] : q.model_actions[rep];
    if (q.met_final)
        for (int j = 0; j < 3; j++) {
            const int64_t a = q.met_in[(int64_t)rep * 3 + j], b = q.met_final[(int64_t)rep * 3 + j];
            if (a > b) q.met_final[(int64_t)rep * 3 + j] = a;
        }
    int4 out = make_int4(0, 0, 0, 0);
    if (d[MARO_DEC_STATUS] == MARO_STATUS_DECISION) {
        const int tick = d[MARO_DEC_TICK], vessel = d[MARO_DEC_VESSEL];
        int m = q.model_actions_i64 ? (int)q.model_actions_i64[rep] : q.model_actions[rep];
        m = m < 0 ? 0 : (m >= q.n_action_space ? q.n_action_space - 1 : m);
        const int32_t* now = nullptr;
        const bool have_now = snap_row(q, rep, tick, now);
        const double percent = fabs(q.action_space[m]);
        const double zero_action_idx = (double)q.n_action_space / 2.0;
        double quantity;
        int type;
        if ((double)m < zero_action_idx) {
            type = 0;  // ActionType.LOAD
            quantity = rint(percent * (double)d[MARO_DEC_SCOPE_LOAD]);  // python round(): half to even
            if (q.finite_vessel_space) {
                const double space = have_now ? (double)now[q.off_remaining_space + vessel] : 0.0;
                quantity = quantity <= space ? quantity : space;
            }
        } else {
            type = 1;  // ActionType.DISCHARGE ((double)m == zero_action_idx cannot happen for an odd-sized space either way)
            const double early = q.has_early_discharge && have_now ? (double)now[q.off_early_discharge + vessel] : 0.0;
            const double plan = percent * ((double)d[MARO_DEC_SCOPE_DISCHARGE] + early) - early;
            quantity = plan > 0 ? rint(plan) : rint(percent * (double)d[MARO_DEC_SCOPE_DISCHARGE]);
        }
        out = make_int4(vessel, d[MARO_DEC_PORT], (int)quantity, type);
    }
    *reinterpret_cast<int4*>(q.actions_out + (int64_t)rep * q.max_actions * 4) = out;
}

static int shape_common(MaroCimEnv* e, ShapeArgs& q) {
    memset(&q, 0, sizeof(q));
    q.snap = e->d_snap; q.snap_frame = e->d_snap_frame; q.ring_rows = e->ring_rows; q.FWp = e->FWp; q.B = e->B;
    q.P = e->s.P; q.V = e->s.V; q.o_fut = e->s.o_fut; q.fut = e->s.fut;
    return 0;
}

extern "C" {

int32_t maro_cim_rl_state_dim(MaroCimEnv* e, int32_t look_back, int32_t n_port_attrs, int32_t n_vessel_attrs) {
    if (!e || look_back < 2) return -1;
    return (look_back - 1) * (1 + e->s.fut) * n_port_attrs + n_vessel_attrs;
}

static int rl_state_launch(MaroCimEnv* e, const int32_t* d_decisions, int32_t look_back, const int32_t* port_attrs, int32_t n_port_attrs,
                           const int32_t* vessel_attrs, int32_t n_vessel_attrs, double* d_out, float* d_out_f32) {
    if (!e || !d_decisions || (!d_out && !d_out_f32) || !port_attrs || !vessel_attrs || look_back < 2 || n_port_attrs < 1 ||
        n_port_attrs > 16 || n_vessel_attrs < 0 || n_vessel_attrs > 16)
        return fail("maro_cim_rl_state_device: bad arguments");
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    ShapeArgs q;
    shape_common(e, q);
    for (int i = 0; i < n_port_attrs; i++) {
        int a = port_attrs[i];
        if (a < 0 || a >= (int)e->attrs[0].size() || e->attrs[0][a].slots != 1) return fail("maro_cim_rl_state_device: bad port attribute");
        q.port_attr_off[i] = e->attrs[0][a].off; q.port_attr_isf[i] = e->attrs[0][a].isf;
    }
    for (int i = 0; i < n_vessel_attrs; i++) {
        int a = vessel_attrs[i];
        if (a < 0 || a >= (int)e->attrs[1].size() || e->attrs[1][a].slots != 1) return fail("maro_cim_rl_state_device: bad vessel attribute");
        q.vessel_attr_off[i] = e->attrs[1][a].off; q.vessel_attr_isf[i] = e->attrs[1][a].isf;
    }
    q.decisions = d_decisions; q.look_back_ticks = look_back - 1; q.n_ports_per_state = 1 + e->s.fut;
    q.npa = n_port_attrs; q.nva = n_vessel_attrs; q.state_out = d_out; q.state_out_f32 = d_out_f32;
    const int64_t total = (int64_t)e->B * maro_cim_rl_state_dim(e, look_back, n_port_attrs, n_vessel_attrs);
    int threads = 256, blocks = (int)std::min<int64_t>((total + threads - 1) / threads, (int64_t)e->n_sm * 8);
    cim_rl_state_kernel<<<blocks, threads, 0, e->stream>>>(q);
    CK(cudaGetLastError());
    return 0;
}

int maro_cim_rl_state_device(MaroCimEnv* e, const int32_t* d_decisions, int32_t look_back, const int32_t* port_attrs,
                             int32_t n_port_attrs, const int32_t* vessel_attrs, int32_t n_vessel_attrs, double* d_out) {
    if (!d_out) return fail("maro_cim_rl_state_device: bad arguments");
    return rl_state_launch(e, d_decisions, look_back, port_attrs, n_port_attrs, vessel_attrs, n_vessel_attrs, d_out, nullptr);
}

int maro_cim_rl_state_f32_device(MaroCimEnv* e, const int32_t* d_decisions, int32_t look_back, const int32_t* port_attrs,
                                 int32_t n_port_attrs, const int32_t* vessel_attrs, int32_t n_vessel_attrs, float* d_out) {
    if (!d_out) return fail("maro_cim_rl_state_f32_device: bad arguments");
    return rl_state_launch(e, d_decisions, look_back, port_attrs, n_port_attrs, vessel_attrs, n_vessel_attrs, nullptr, d_out);
}

static int rl_action_launch(MaroCimEnv* e, ShapeArgs& q, const int32_t* d_decisions, const double* d_action_space, int32_t n_action_space,
                            int32_t finite_vessel_space, int32_t has_early_discharge, int32_t* d_actions) {
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    q.decisions = d_decisions; q.action_space = d_action_space; q.n_action_space = n_action_space;
    q.finite_vessel_space = finite_vessel_space; q.has_early_discharge = has_early_discharge; q.max_actions = e->s.max_actions;
    q.off_remaining_space = e->attrs[1][common_attr_id(e, 1, "remaining_space")].off;
    q.off_early_discharge = e->attrs[1][common_attr_id(e, 1, "early_discharge")].off;
    q.actions_out = d_actions;
    int threads = 256, blocks = (e->B + threads - 1) / threads;
    cim_rl_action_kernel<<<blocks, threads, 0, e->stream>>>(q);
    CK(cudaGetLastError());
    return 0;
}

int maro_cim_rl_action_device(MaroCimEnv* e, const int32_t* d_decisions, const int32_t* d_model_actions, const double* d_action_space,
                              int32_t n_action_space, int32_t finite_vessel_space, int32_t has_early_discharge, int32_t* d_actions) {
    if (!e || !d_decisions || !d_model_actions || !d_action_space || !d_actions || n_action_space < 1)
        return fail("maro_cim_rl_action_device: bad arguments");
    ShapeArgs q;
    shape_common(e, q);
    q.model_actions = d_model_actions;
    return rl_action_launch(e, q, d_decisions, d_action_space, n_action_space, finite_vessel_space, has_early_discharge, d_actions);
}

int maro_cim_rl_action_ex_device(MaroCimEnv* e, const int32_t* d_decisions, const void* d_model_actions, int32_t model_actions_are_i64,
                                 int32_t* d_model_actions_record, const int64_t* d_metrics_in, int64_t* d_metrics_final,
                                 const double* d_action_space, int32_t n_action_space, int32_t finite_vessel_space,
                                 int32_t has_early_discharge, int32_t* d_actions) {
    if (!e || !d_decisions || !d_model_actions || !d_action_space || !d_actions || n_action_space < 1 || (!d_metrics_in) != (!d_metrics_final))
        return fail("maro_cim_rl_action_ex_device: bad arguments");
    ShapeArgs q;
    shape_common(e, q);
    if (model_actions_are_i64) q.model_actions_i64 = static_cast<const int64_t*>(d_model_actions);
    else q.model_actions = static_cast<const int32_t*>(d_model_actions);
    q.model_actions_record = d_model_actions_record; q.met_in = d_metrics_in; q.met_final = d_metrics_final;
    return rl_action_launch(e, q, d_decisions, d_action_space, n_action_space, finite_vessel_space, has_early_discharge, d_actions);
}

static int rl_reward_launch(MaroCimEnv* e, const int32_t* d_ticks, const int32_t* d_ports, int32_t n_rows, const double* d_decay,
                            int32_t time_window, double fulfillment_factor, double shortage_factor, float* d_out) {
    CK(cudaSetDevice(e->device));
    END_SESSION(e);
    ShapeArgs q;
    shape_common(e, q);
    q.ticks = d_ticks; q.ports = d_ports; q.decay = d_decay; q.time_window = time_window; q.n_rows = n_rows;
    q.off_fulfillment = e->attrs[0][common_attr_id(e, 0, "fulfillment")].off;
    q.off_shortage = e->attrs[0][common_attr_id(e, 0, "shortage")].off;
    q.fulfillment_factor = fulfillment_factor; q.shortage_factor = shortage_factor; q.reward_out = d_out;
    const int64_t items = (int64_t)n_rows * e->B;
    int threads = 128, blocks = (int)std::min<int64_t>((items * 32 + threads - 1) / threads, (int64_t)e->n_sm * 16);
    cim_rl_reward_kernel<<<blocks, threads, 0, e->stream>>>(q);
    CK(cudaGetLastError());
    return 0;
}

int maro_cim_rl_reward_device(MaroCimEnv* e, const int32_t* d_ticks, const int32_t* d_ports, const double* d_decay,
                              int32_t time_window, double fulfillment_factor, double shortage_factor, float* d_out) {
    if (!e || !d_ticks || !d_ports || !d_decay || !d_out || time_window < 1) return fail("maro_cim_rl_reward_device: bad arguments");
    return rl_reward_launch(e, d_ticks, d_ports, 1, d_decay, time_window, fulfillment_factor, shortage_factor, d_out);
}

/* the rewards of a whole trajectory in ONE launch: ticks / ports / out are [n_rows][n_replicas] (row = rollout step) */
int maro_cim_rl_reward_batch_device(MaroCimEnv* e, const int32_t* d_ticks, const int32_t* d_ports, int32_t n_rows, const double* d_decay,
                                    int32_t time_window, double fulfillment_factor, double shortage_factor, float* d_out) {
    if (!e || !d_ticks || !d_ports || !d_decay || !d_out || time_window < 1 || n_rows < 1)
        return fail("maro_cim_rl_reward_batch_device: bad arguments");
    return rl_reward_launch(e, d_ticks, d_ports, n_rows, d_decay, time_window, fulfillment_factor, shortage_factor, d_out);
}

}  // extern "C"

