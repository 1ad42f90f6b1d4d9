// cim_core.cuh — per-replica CIM simulation core (device code; one lane group of G lanes = one replica, G = 32 is
// "one warp = one replica", smaller G packs 32/G replicas of a small topology into a warp).
//
// A from-scratch formulation of the reference's Env.step hot path
// (maro/simulator/core.py:317-381, maro/event_buffer/event_buffer.py:190-247,
//  maro/simulator/scenarios/cim/business_engine.py:122-224, 448-748) for a SIMT machine:
//
//   * The reference keeps one linked list of event objects per tick.  Here the per-tick execution order is
//     reconstructed from its sources (DESIGN.md §4):
//       (a) VESSEL_DEPARTURE events pre-inserted at init  -> read off the static stop table, one lane per vessel,
//       (b) events inserted by earlier ticks (RETURN_FULL / DISCHARGE_FULL / RETURN_EMPTY) -> calendar queue bucket,
//       (c) ORDER events of BusinessEngine.step -> precomputed schedule (noise-free) or generated in place,
//       (d) VESSEL_ARRIVAL + LOAD_FULL per arriving vessel, then (e) the decision events, vessel order.
//   * Every phase is a cooperative group operation: lane i takes the i-th event of the phase.  Order dependence
//     inside a phase is resolved with shuffles / ballots instead of serial execution:
//       - phase (b) handlers are pure adds/subtracts -> shared-memory atomics, any order;
//       - ORDERs of one source port consume `empty` in sequence -> segmented prefix sum over the lanes;
//       - LOAD_FULL hands `acceptable` space to the reachable stops in sequence -> prefix sum over the lanes;
//       - events pushed by several lanes keep FIFO order per target bucket via match_any + lane ranks;
//       - MT19937 draws are indexed by event rank (random access into the stream, parallel twist).
//
// The same source compiles for the host with MARO_HOST_EMULATION (tests/_emul_src: one host thread per lane); that
// build exists only to debug the kernel logic without a GPU and is never part of the shipped library.
#pragma once
#include <stdint.h>

#ifdef MARO_HOST_EMULATION
#include <math.h>
#include <string.h>

#include "warp_emul.hpp"
#define MARO_DEV inline
#else
#define MARO_DEV __device__ __forceinline__
#endif

namespace maro {

// =====================================================================================================
// Lane-group primitives
// =====================================================================================================
#ifdef MARO_HOST_EMULATION
template <int G>
struct Grp {
    int lane;
    explicit Grp(int l) : lane(l) {}
    void sync() const { wemu::barrier(); }
    int shfl(int x, int src) const {
        uint64_t o[32];
        wemu::exchange((uint64_t)(uint32_t)x, o);
        return (int)(uint32_t)o[src & (G - 1)];
    }
    int shfl_up(int x, int d) const {
        uint64_t o[32];
        wemu::exchange((uint64_t)(uint32_t)x, o);
        return lane >= d ? (int)(uint32_t)o[lane - d] : x;
    }
    int shfl_down(int x, int d) const {
        uint64_t o[32];
        wemu::exchange((uint64_t)(uint32_t)x, o);
        return lane + d < G ? (int)(uint32_t)o[lane + d] : x;
    }
    uint32_t ballot(bool p) const {
        uint64_t o[32];
        wemu::exchange(p ? 1 : 0, o);
        uint32_t m = 0;
        for (int i = 0; i < G; i++) m |= (uint32_t)o[i] << i;
        return m;
    }
    uint32_t match(int v) const {
        uint64_t o[32];
        wemu::exchange((uint64_t)(uint32_t)v, o);
        uint32_t m = 0;
        for (int i = 0; i < G; i++) if ((uint32_t)o[i] == (uint32_t)v) m |= 1u << i;
        return m;
    }
    int64_t sum64(int64_t x) const {
        uint64_t o[32];
        wemu::exchange((uint64_t)x, o);
        int64_t s = 0;
        for (int i = 0; i < G; i++) s += (int64_t)o[i];
        return s;
    }
    int sum(int x) const { return (int)sum64(x); }
    uint32_t or32(uint32_t x) const {
        uint64_t o[32];
        wemu::exchange(x, o);
        uint32_t m = 0;
        for (int i = 0; i < G; i++) m |= (uint32_t)o[i];
        return m;
    }
};
static inline void atomic_add(int32_t* p, int32_t v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline double maro_ceil(double x) { return ceil(x); }
static inline double maro_floor(double x) { return floor(x); }
static inline float maro_d2f(double x) { return (float)x; }
static inline int32_t maro_f2i(float x) { int32_t i; memcpy(&i, &x, 4); return i; }
static inline float maro_i2f(int32_t i) { float x; memcpy(&x, &i, 4); return x; }
static inline int maro_ffs64(uint64_t x) { return __builtin_ffsll((long long)x); }
static inline int maro_ffs32(uint32_t x) { return __builtin_ffs((int)x); }
static inline int maro_popc(uint32_t x) { return __builtin_popcount(x); }
static inline int maro_clz(uint32_t x) { return x ? __builtin_clz(x) : 32; }
#else
template <int G>
struct Grp {
    int lane;       // 0..G-1 inside the group
    unsigned mask;  // lanes of this group inside the warp
    int base;
    __device__ __forceinline__ explicit Grp(int lane_in_warp) {
        lane = lane_in_warp & (G - 1);
        base = lane_in_warp & ~(G - 1);
        mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << base);
    }
    __device__ __forceinline__ void sync() const { __syncwarp(mask); }
    __device__ __forceinline__ int shfl(int x, int src) const { return __shfl_sync(mask, x, src, G); }
    __device__ __forceinline__ int shfl_up(int x, int d) const { return __shfl_up_sync(mask, x, d, G); }
    __device__ __forceinline__ int shfl_down(int x, int d) const { return __shfl_down_sync(mask, x, d, G); }
    __device__ __forceinline__ uint32_t ballot(bool p) const {
        uint32_t b = __ballot_sync(mask, p);
        return G == 32 ? b : ((b >> base) & ((1u << G) - 1u));
    }
    __device__ __forceinline__ uint32_t match(int v) const {
        uint32_t b = __match_any_sync(mask, v);
        return G == 32 ? b : ((b >> base) & ((1u << G) - 1u));
    }
    __device__ __forceinline__ int64_t sum64(int64_t x) const {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) x += __shfl_xor_sync(mask, x, o, G);
        return x;
    }
    __device__ __forceinline__ int sum(int x) const {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) x += __shfl_xor_sync(mask, x, o, G);
        return x;
    }
    __device__ __forceinline__ uint32_t or32(uint32_t x) const {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) x |= __shfl_xor_sync(mask, x, o, G);
        return x;
    }
};
__device__ __forceinline__ void atomic_add(int32_t* p, int32_t v) { atomicAdd(p, v); }
__device__ __forceinline__ double maro_ceil(double x) { return ceil(x); }
__device__ __forceinline__ double maro_floor(double x) { return floor(x); }
__device__ __forceinline__ float maro_d2f(double x) { return __double2float_rn(x); }
__device__ __forceinline__ int32_t maro_f2i(float x) { return __float_as_int(x); }
__device__ __forceinline__ float maro_i2f(int32_t i) { return __int_as_float(i); }
__device__ __forceinline__ int maro_ffs64(uint64_t x) { return __ffsll((long long)x); }
__device__ __forceinline__ int maro_ffs32(uint32_t x) { return __ffs((int)x); }
__device__ __forceinline__ int maro_popc(uint32_t x) { return __popc(x); }
__device__ __forceinline__ int maro_clz(uint32_t x) { return __clz((int)x); }
#endif

#define LANE_LOOP(i, n) for (int i = g.lane; i < (n); i += G)
// loop over a topology dimension (ports, vessels, ...): groups narrower than a warp are sized >= every such dimension
// (lanes_per_replica), so the loop is a single predicated pass there
#ifdef MARO_HOST_EMULATION  // the tests also run widths narrower than the topology to exercise every chunk loop
#define LANE_DIM(i, n) LANE_LOOP(i, n)
#else
#define LANE_DIM(i, n) for (int i = g.lane; i < (n); i += (G < 32 ? 0x40000000 : G))
#endif

// chunks of G over a topology dimension that every lane group of the small-topology instantiation covers in one pass
// (kSmall: P, V, route lengths and fut are <= G): a constant trip count of one there
#define GROUP_CHUNKS(b0, n) for (int b0 = 0; b0 < (kSmall ? 1 : (n)); b0 += G)

// inclusive prefix sum over the lanes of a group
template <int G>
MARO_DEV int scan_incl(const Grp<G>& g, int x) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) {
        int t = g.shfl_up(x, d);
        if (g.lane >= d) x += t;
    }
    return x;
}

// inclusive prefix sum restricted to runs of equal `key` (keys sorted / contiguous)
template <int G>
MARO_DEV int scan_incl_seg(const Grp<G>& g, int x, int key) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) {
        int t = g.shfl_up(x, d);
        int k = g.shfl_up(key, d);
        if (g.lane >= d && k == key) x += t;
    }
    return x;
}

// ---------------------------------------------------------------------------------------------------
// Shape / layout shared by every replica of a handle (kernel parameter; offsets are in 4-byte words).
// ---------------------------------------------------------------------------------------------------
enum PortAttr { PA_ACC_BOOKING, PA_ACC_FULFILLMENT, PA_ACC_SHORTAGE, PA_BOOKING, PA_CAPACITY, PA_EMPTY,
                PA_FULFILLMENT, PA_FULL, PA_ON_CONSIGNEE, PA_ON_SHIPPER, PA_SHORTAGE, PA_TRANSFER_COST, PA_COUNT };
enum VesselAttr { VA_CAPACITY, VA_EARLY_DISCHARGE, VA_EMPTY, VA_FULL, VA_IS_PARKING, VA_LAST_LOC_IDX,
                  VA_LOC_PORT_IDX, VA_NEXT_LOC_IDX, VA_REMAINING_SPACE, VA_ROUTE_IDX, VA_COUNT };

// control words (per replica, after the frame)
enum Ctrl {
    C_STATE, C_TICK, C_ARR_LO, C_ARR_HI, C_DEC_POS, C_FREE_TOP, C_Q_COUNT, C_ERR,
    C_OPNUM_LO, C_OPNUM_HI, C_MT_ORDER_IDX, C_MT_BUFFER_IDX,
    C_NSTEPS_LO, C_NSTEPS_HI, C_NTICKS_LO, C_NTICKS_HI, C_NEVENTS_LO, C_NEVENTS_HI, C_NSNAPS_LO, C_NSNAPS_HI,
    C_LAST_FRAME, C_N_ORDERS, C_EP_STEP, C_RESERVED2,
    C_FIXED  // followed by dep_cursor[V], next_dep_tick[V], next_arr_tick[V] (+ due_stop[V], due_tick[V] with due rings)
};
#define NO_TICK 0x7fffffff
enum State { ST_START = 0, ST_TICK_BEGIN = 1, ST_DECISIONS = 2, ST_AWAIT = 3, ST_DONE = 4, ST_FINISHED = 5, ST_ERROR = 6 };
enum DynEv { DE_RETURN_FULL = 0, DE_DISCHARGE_FULL = 1, DE_RETURN_EMPTY = 2 };

struct CimShape {
    int P, V, R, past, fut, max_route_len;
    int max_tick, start_tick, resolution, ring_rows, order_mode, total_containers;
    int order_noise, buffer_noise, max_actions, n_replicas;
    int vol_is_one, max_targets;
    int res_is_one;  // snapshot_resolution == 1 (skips the per-tick integer divisions)
    double vol;
    // per-replica state block: [frame FWp][ctrl CWp][queue: ev QN*2 | buckets QH | next+free u16 QN]
    int FW, FWp, CWp, QN, QH, SW;
    int o_vs, o_past, o_past_tick, o_fut, o_fut_tick, o_fop, o_fov, o_vp;  // frame offsets (ports start at 0)
    // static table blob offsets (words from the blob start); *_d are offsets of double arrays (even)
    int t_port_capacity, t_port_init_empty, t_frb_d, t_frn_d, t_erb_d, t_ern_d, t_sb_d, t_sn_d;
    int t_target_offset, t_target_port, t_tb_d, t_tn_d;
    int t_vessel_capacity, t_vessel_init_empty, t_vessel_route, t_vessel_period, t_vessel_route_start;
    int t_vessel_leg_offset, t_vessel_leg, t_stop_offset, t_stop_arrival, t_stop_leave, t_stop_port;
    int t_route_offset, t_route_port, t_order_proportion, t_mt_order, t_mt_buffer;
    // precomputed schedules for noise-free topologies (0 offsets when unused)
    int order_table;                        // 1: per-tick order lists are static (fixed mode, no order noise)
    int t_ord_slot, t_ord_off, t_ord_list;  // slot[max_tick] -> off[slot..slot+1] -> list {src | dst << 8, qty}
    int t_frb_i, t_erb_i;                   // ceil(buffer_ticks) per port, valid when buffer_noise == 0
    int table_words;                        // stride between topology blobs
    int mt_scratch;                         // word offset of the scratch area inside a replica's MT block
    // Delay lines (noise-free topologies with few ports; 0 = off): RETURN_FULL / RETURN_EMPTY fire a fixed, small number
    // of ticks after they are created and are pure adds, so they are ACCUMULATED per due tick instead of queued as events:
    // slot (tick & (DL-1)) = { rf[P*P] (src*P+dst -> quantity), re[P] (port -> quantity), n_rf, n_re (event counts) } at word
    // offset o_dl of the state block.  Same arithmetic, same event counts, no list walking / free list / push machinery.
    int DL, o_dl, dl_stride;
    // Due rings (delay-line handles whose every vessel visits its stops at strictly increasing ticks; 0 = off, the calendar
    // queue carries DISCHARGE_FULL): the discharges LOAD_FULL schedules are pure adds due at a known stop of the loading vessel,
    // so they are ACCUMULATED per (vessel, stop) instead of queued: vessel v's ring of due_R slots {quantity, events} at word
    // offset o_due + 2 * due_R * v, slot = stop index & (due_R - 1), due_R = power of two > max_route_len.  The control
    // block holds each vessel's next due stop and its arrival tick (C_FIXED + 3V + v, + 4V + v; kSmall: Ctl on lane v).
    int due_R, o_due;
    // DecisionMode.Joint (core.py:354-366): every decision event of a tick is returned at once (V rows of 8 words), the
    // answers are applied in list order when the replica is stepped again.  DW = words of a replica's decision block.
    int joint, DW;
};

// ---------------------------------------------------------------------------------------------------
// Per-phase cycle attribution of the step's dependent chain, compiled in only with -DMARO_PHASE_CLOCKS (tools/phase_clocks.py
// builds that variant).  PHASE_MARK(r, ph) charges the cycles since the previous mark to phase `ph`; the resident rollout keeps
// the accumulators in registers and adds them to maro_phase_clk once per launch.
// ---------------------------------------------------------------------------------------------------
enum Phase { PH_AGENT, PH_ACTIONS, PH_VESSELS, PH_BUCKET, PH_DELAY, PH_ORDERS, PH_ARRIVALS, PH_DECISION, PH_POST, PH_STORE,
             PH_COUNT, PH_STEPS = PH_COUNT, PH_TICKS, PH_SLOTS };
#if defined(MARO_PHASE_CLOCKS) && !defined(MARO_HOST_EMULATION)
struct PhaseClk {
    long long t;                   // clock64() at the previous mark
    unsigned long long acc[PH_SLOTS];  // cycles per phase, then env-steps and ticks
};
#define PHASE_MARK(r, ph)                              \
    do {                                               \
        if ((r).pc) {                                  \
            const long long _t = clock64();            \
            (r).pc->acc[ph] += (unsigned long long)(_t - (r).pc->t); \
            (r).pc->t = _t;                            \
        }                                              \
    } while (0)
#define PHASE_COUNT(r, slot, n) do { if ((r).pc) (r).pc->acc[slot] += (unsigned long long)(n); } while (0)
#else
#define PHASE_MARK(r, ph) do {} while (0)
#define PHASE_COUNT(r, slot, n) do {} while (0)
#endif

struct Replica {
    int32_t* f;          // frame words (shared memory on the device)
    int32_t* c;          // control words
    int32_t* q;          // queue: pool | buckets | free stack
    const int32_t* t;    // static table blob of this replica's topology
    uint32_t* mt;        // [2][640] MT19937 states + scratch, global memory (NULL when the topology has no noise)
    int32_t* snap;       // [ring_rows][FWp] snapshot ring (global)
    int32_t* snap_frame; // [ring_rows] frame index held by each row
#if defined(MARO_PHASE_CLOCKS) && !defined(MARO_HOST_EMULATION)
    PhaseClk* pc;        // phase accumulators of this lane (resident rollouts only, else NULL)
#endif
};

#define TBL_I(r, off, i) ((r).t[(off) + (i)])
#define TBL_D(r, off, i) (reinterpret_cast<const double*>((r).t + (off))[(i)])

MARO_DEV int32_t& PA(const CimShape& s, const Replica& r, int attr, int p) { return r.f[attr * s.P + p]; }
MARO_DEV int32_t& VA(const CimShape& s, const Replica& r, int attr, int v) { return r.f[s.o_vs + attr * s.V + v]; }

// 64-bit control words sit on even word indices of a 16-byte aligned block: one 64-bit access each
MARO_DEV int64_t ctrl_get64(const Replica& r, int lo) { return *reinterpret_cast<const int64_t*>(r.c + lo); }
MARO_DEV void ctrl_set64(const Replica& r, int lo, int64_t v) { *reinterpret_cast<int64_t*>(r.c + lo) = v; }
MARO_DEV void ctrl_add64(const Replica& r, int lo, int64_t d) { ctrl_set64(r, lo, ctrl_get64(r, lo) + d); }

// ------------------------------------------------------------------------------------------------
// Control state that replica_step reads or writes on every step, held in registers for as long as the block stays on the SM
// (a resident launch: loaded once after stage-in, stored once before write-back; other callers around each call).  The
// scalars are the same in every lane of the group; the 64-bit counters are kept by the leader lane.  In the small-topology
// instantiation (kSmall: V <= G) lane v also holds vessel v's five cursors C_FIXED + {0, V, 2V, 3V, 4V} + v.  What stays in
// the control block (free stack top, error word, MT19937 positions, ...) is shared-memory state of the phases that use it.
// ------------------------------------------------------------------------------------------------
struct Ctl {
    int state, tick, dec_pos, ep_step, last_frame;
    uint64_t arr;  // vessels arriving this tick (C_ARR_LO / C_ARR_HI)
    int64_t opnum, nsteps, nticks, nevents, nsnaps;
    int64_t ndue;  // events the due rings executed on THIS lane (per-lane partial count, added to C_NEVENTS by ctl_store)
    int dep_cursor, next_dep, next_arr;  // kSmall: vessel g.lane's cursors (NO_TICK on lanes >= V)
    int due_stop, due_tick;              // kSmall: vessel g.lane's next due stop and its arrival tick (NO_TICK on lanes >= V)
    bool snap_pending;  // deferred pre-decision snapshot not written yet (fused rollouts, replica_step<..., kDeferSnap>)
};

template <int G, bool kSmall>
MARO_DEV void ctl_load(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k) {
    k.ndue = 0;
    k.snap_pending = false;
    k.state = r.c[C_STATE];
    k.tick = r.c[C_TICK];
    k.dec_pos = r.c[C_DEC_POS];
    k.ep_step = r.c[C_EP_STEP];
    k.last_frame = r.c[C_LAST_FRAME];
    k.arr = ((uint64_t)(uint32_t)r.c[C_ARR_HI] << 32) | (uint32_t)r.c[C_ARR_LO];
    k.opnum = ctrl_get64(r, C_OPNUM_LO);
    k.nsteps = ctrl_get64(r, C_NSTEPS_LO);
    k.nticks = ctrl_get64(r, C_NTICKS_LO);
    k.nevents = ctrl_get64(r, C_NEVENTS_LO);
    k.nsnaps = ctrl_get64(r, C_NSNAPS_LO);
    const int v = g.lane;
    const bool in = kSmall && v < s.V;
    k.dep_cursor = in ? r.c[C_FIXED + v] : 0;
    k.next_dep = in ? r.c[C_FIXED + s.V + v] : NO_TICK;
    k.next_arr = in ? r.c[C_FIXED + 2 * s.V + v] : NO_TICK;
    k.due_stop = in ? r.c[C_FIXED + 3 * s.V + v] : 0;
    k.due_tick = in ? r.c[C_FIXED + 4 * s.V + v] : NO_TICK;
}

// (ends with a group barrier: the control block is complete for every lane afterwards)
template <int G, bool kSmall>
MARO_DEV void ctl_store(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k) {
    const int64_t ndue = g.sum64(k.ndue);
    k.nevents += ndue;  // (every lane: the partials restart from zero)
    k.ndue = 0;
    g.sync();
    if (g.lane == 0) {
        r.c[C_STATE] = k.state;
        r.c[C_TICK] = k.tick;
        r.c[C_DEC_POS] = k.dec_pos;
        r.c[C_EP_STEP] = k.ep_step;
        r.c[C_LAST_FRAME] = k.last_frame;
        r.c[C_ARR_LO] = (int32_t)(uint32_t)(k.arr & 0xffffffffu);
        r.c[C_ARR_HI] = (int32_t)(uint32_t)(k.arr >> 32);
        ctrl_set64(r, C_OPNUM_LO, k.opnum);
        ctrl_set64(r, C_NSTEPS_LO, k.nsteps);
        ctrl_set64(r, C_NTICKS_LO, k.nticks);
        ctrl_set64(r, C_NEVENTS_LO, k.nevents);
        ctrl_set64(r, C_NSNAPS_LO, k.nsnaps);
    }
    const int v = g.lane;
    if (kSmall && v < s.V) {
        r.c[C_FIXED + v] = k.dep_cursor;
        r.c[C_FIXED + s.V + v] = k.next_dep;
        r.c[C_FIXED + 2 * s.V + v] = k.next_arr;
        r.c[C_FIXED + 3 * s.V + v] = k.due_stop;
        r.c[C_FIXED + 4 * s.V + v] = k.due_tick;
    }
    g.sync();
}

// ------------------------------------------------------------------------------------------------
// MT19937, bit-compatible with CPython's random.Random (Modules/_randommodule.c).
// State words live in global memory: r.mt[stream * 640 + i]; scratch (for the stream tail) at r.mt + mt_scratch.
// ------------------------------------------------------------------------------------------------
MARO_DEV uint32_t mt_temper(uint32_t y) {
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}
MARO_DEV uint32_t mt_mix(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

// serial generator step (leader lane only) — used by the noisy order generator
MARO_DEV uint32_t mt_next(const Replica& r, int stream) {
    uint32_t* mt = r.mt + stream * 640;
    int idx = r.c[C_MT_ORDER_IDX + stream];
    if (idx >= 624) {
        int kk;
        for (kk = 0; kk < 624 - 397; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk + 397]);
        for (; kk < 623; kk++) mt[kk] = mt_mix(mt[kk], mt[kk + 1], mt[kk - 227]);
        mt[623] = mt_mix(mt[623], mt[0], mt[396]);
        idx = 0;
    }
    uint32_t y = mt[idx++];
    r.c[C_MT_ORDER_IDX + stream] = idx;
    return mt_temper(y);
}

MARO_DEV double mt_uniform01(uint32_t y0, uint32_t y1) {
    uint32_t a = y0 >> 5, b = y1 >> 6;
    return ((double)a * 67108864.0 + (double)b) * (1.0 / 9007199254740992.0);
}

// value + random.uniform(-noise, noise)   (maro/data_lib/cim/utils.py:30-42; Lib/random.py uniform)
MARO_DEV double noised(double value, double noise, double u) {
    double lo = -noise, hi = noise;
    return value + (lo + (hi - lo) * u);
}
MARO_DEV double apply_noise_serial(const Replica& r, int stream, double value, double noise) {
    uint32_t y0 = mt_next(r, stream), y1 = mt_next(r, stream);
    return noised(value, noise, mt_uniform01(y0, y1));
}

// Cooperative twist of the whole state (all lanes of the group).
template <int G>
MARO_DEV void mt_twist(const Grp<G>& g, uint32_t* mt) {
    for (int b0 = 0; b0 < 623; b0 += G) {
        int kk = b0 + g.lane;
        uint32_t nv = 0;
        if (kk < 623) nv = mt_mix(mt[kk], mt[kk + 1], kk < 227 ? mt[kk + 397] : mt[kk - 227]);
        g.sync();
        if (kk < 623) mt[kk] = nv;
        g.sync();
        // a batch never straddles the 227 boundary dependency: element kk >= 227 reads mt[kk-227] written >= one
        // batch earlier because G <= 32 < 227.
    }
    if (g.lane == 0) mt[623] = mt_mix(mt[623], mt[0], mt[396]);
    g.sync();
}

// Make the next `n_out` tempered outputs of `stream` addressable by rank: output k is view.at(k).
struct MtView {
    const uint32_t* a;
    int na;
    const uint32_t* b;
    MARO_DEV uint32_t at(int k) const { return mt_temper(k < na ? a[k] : b[k - na]); }
};
template <int G>
MARO_DEV MtView mt_reserve(const CimShape& s, const Grp<G>& g, const Replica& r, int stream, int n_out) {
    uint32_t* mt = r.mt + stream * 640;
    int idx = r.c[C_MT_ORDER_IDX + stream];
    MtView v;
    if (idx + n_out <= 624) {
        v.a = mt + idx; v.na = n_out; v.b = mt;
        g.sync();
        if (g.lane == 0) r.c[C_MT_ORDER_IDX + stream] = idx + n_out;
        g.sync();
        return v;
    }
    int tail = 624 - idx;
    uint32_t* scratch = r.mt + s.mt_scratch;
    LANE_LOOP(i, tail) scratch[i] = mt[idx + i];
    g.sync();
    mt_twist(g, mt);
    v.a = scratch; v.na = tail; v.b = mt;
    if (g.lane == 0) r.c[C_MT_ORDER_IDX + stream] = n_out - tail;
    g.sync();
    return v;
}

// ------------------------------------------------------------------------------------------------
// Calendar queue of dynamic events.  Slot = 2 words {type|a<<8|b<<16|c<<24, qty} + a 16-bit next link;
// bucket[tick & (QH-1)] = head | tail << 16 (0xffff = nil); free slots on a 16-bit stack (parallel pop / push).
// Layout inside the replica's queue region: ev[QN][2] | bucket[QH] | nxt[QN] (u16) | free[QN] (u16).
// group_push: every lane with `want` appends one event; FIFO order per bucket = lane order.
// ------------------------------------------------------------------------------------------------
#define Q_NIL 0xffff
MARO_DEV int32_t* q_bucket(const CimShape& s, const Replica& r) { return r.q + s.QN * 2; }
MARO_DEV uint16_t* q_next(const CimShape& s, const Replica& r) { return reinterpret_cast<uint16_t*>(r.q + s.QN * 2 + s.QH); }
MARO_DEV uint16_t* q_free(const CimShape& s, const Replica& r) { return q_next(s, r) + s.QN; }

MARO_DEV int32_t* dl_slot(const CimShape& s, const Replica& r, int tick) { return r.f + s.o_dl + (tick & (s.DL - 1)) * s.dl_stride; }

// Due-ring slot {quantity, events} of vessel v's stop `stop`.  No two outstanding stops of a vessel share a slot: LOAD_FULL at
// stop `loc` schedules discharges at stops loc + 1 .. loc + rl only (rl = the vessel's route length), and the drain cursor has
// passed every stop up to the vessel's latest arrival (stop ticks increase strictly, the drain of tick T runs before that
// tick's arrivals).  So the outstanding stops of a vessel lie in (loc, loc + rl] for its latest arrival stop loc -- at most
// rl < due_R consecutive stop indices.
MARO_DEV int32_t* due_slot(const CimShape& s, const Replica& r, int v, int stop) {
    return r.f + s.o_due + 2 * (v * s.due_R + (stop & (s.due_R - 1)));
}

// Phase (b) for the due rings, vessel v (one lane): the DISCHARGE_FULL events (:658-693) accumulated for its stop `stop`,
// due at `tick`, and the RETURN_EMPTY each of them creates -- the arithmetic of run_bucket's discharge branch on the summed
// quantity.  Immediate returns (empty-return buffer 0) cancel on on_consignee.  Returns the events executed.
MARO_DEV int drain_due_stop(const CimShape& s, const Replica& r, int v, int stop, int tick) {
    int32_t* sl = due_slot(s, r, v, stop);
    const int n = sl[1];
    if (n == 0) return 0;
    const int qty = sl[0];
    sl[0] = 0;
    sl[1] = 0;
    const int port = TBL_I(r, s.t_stop_port, TBL_I(r, s.t_stop_offset, v) + stop);
    VA(s, r, VA_FULL, v) -= qty;
    VA(s, r, VA_REMAINING_SPACE, v) += qty;
    r.f[s.o_fov + v * s.P + port] -= qty;
    const int buf = TBL_I(r, s.t_erb_i, port);
    if (buf == 0) {
        atomic_add(&PA(s, r, PA_EMPTY, port), qty);
        return 2 * n;
    }
    atomic_add(&PA(s, r, PA_ON_CONSIGNEE, port), qty);
    if (tick + buf < s.max_tick) {
        int32_t* dl = dl_slot(s, r, tick + buf);
        atomic_add(&dl[s.P * s.P + port], qty);
        atomic_add(&dl[s.P * s.P + s.P + 1], n);
    }
    return n;
}

// Drain the delay-line slot of `tick`: every accumulated RETURN_FULL (:499-522) and RETURN_EMPTY (:695-706) of this tick.
// kSmall (P <= G): lane p drains source port p's row and port p's RETURN_EMPTY entry, then applies the row's total to port p
// -- the same integer sums with plain updates of the lane's own port instead of shared-memory atomics on shared ports.
template <int G, bool kSmall>
MARO_DEV int run_delay_line(const CimShape& s, const Grp<G>& g, const Replica& r, int tick) {
    int32_t* sl = dl_slot(s, r, tick);
    const int PP = s.P * s.P;
    const int n = sl[PP + s.P] + sl[PP + s.P + 1];
    if (n == 0) return 0;  // group-uniform
    g.sync();
    if (kSmall) {
        const int p = g.lane;
        if (p < s.P) {
            int32_t* row = sl + p * s.P;
            int32_t* fop = r.f + s.o_fop + p * s.P;
            int tot = 0;
            for (int d = 0; d < s.P; d++) {
                const int q = row[d];
                if (q) { fop[d] += q; row[d] = 0; tot += q; }
            }
            if (tot) {
                PA(s, r, PA_ON_SHIPPER, p) -= tot;
                PA(s, r, PA_FULL, p) += tot;
            }
            const int qe = sl[PP + p];
            if (qe) {
                PA(s, r, PA_ON_CONSIGNEE, p) -= qe;
                PA(s, r, PA_EMPTY, p) += qe;
                sl[PP + p] = 0;
            }
        }
        if (g.lane == 0) { sl[PP + s.P] = 0; sl[PP + s.P + 1] = 0; }  // (every lane read them above the barrier)
        g.sync();
        return n;
    }
    int src = g.lane / s.P, dst = g.lane - src * s.P;
    for (int i = g.lane; i < PP; i += G) {
        const int q = sl[i];
        if (q) {
            atomic_add(&PA(s, r, PA_ON_SHIPPER, src), -q);
            atomic_add(&PA(s, r, PA_FULL, src), q);
            r.f[s.o_fop + i] += q;
            sl[i] = 0;
        }
        dst += G;
        while (dst >= s.P) { dst -= s.P; src++; }
    }
    g.sync();  // (on_consignee / empty below are plain updates of the lane's own port)
    LANE_DIM(p, s.P) {
        const int q = sl[PP + p];
        if (q) {
            PA(s, r, PA_ON_CONSIGNEE, p) -= q;
            PA(s, r, PA_EMPTY, p) += q;
            sl[PP + p] = 0;
        }
    }
    g.sync();
    if (g.lane == 0) { sl[PP + s.P] = 0; sl[PP + s.P + 1] = 0; }
    g.sync();
    return n;
}

#if defined(MARO_HOST_EMULATION) && defined(MARO_TRACK_QPEAK)
extern "C" int maro_emul_qpeak;
#endif
template <int G>
MARO_DEV void group_push(const CimShape& s, const Grp<G>& g, const Replica& r, bool want, int now, int tick, int w0, int qty) {
    want = want && tick < s.max_tick && tick >= 0;  // later ticks are never visited by the Env (event_buffer.py:190)
    uint32_t bal = g.ballot(want);
    if (bal == 0) return;
    if (g.ballot(want && tick - now >= s.QH)) {  // beyond the calendar horizon the bucket would alias: never silently
        g.sync();
        if (g.lane == 0) r.c[C_ERR] = -2;
        g.sync();
        return;
    }
    int n = maro_popc(bal);
    int rank = maro_popc(bal & ((1u << g.lane) - 1u));
    int top = r.c[C_FREE_TOP];
    if (top < n) {  // group-uniform
        g.sync();
        if (g.lane == 0) r.c[C_ERR] = -2;
        g.sync();
        return;
    }
    uint16_t* fs = q_free(s, r);
    uint16_t* nx = q_next(s, r);
    int slot = want ? fs[top - 1 - rank] : Q_NIL;
    int b = tick & (s.QH - 1);
    uint32_t peers = g.match(want ? b : (0x10000 + g.lane));
    uint32_t below = peers & ((1u << g.lane) - 1u);
    uint32_t above = g.lane == 31 ? 0u : (peers & ~((2u << g.lane) - 1u));
    int nxt_lane = above ? maro_ffs32(above) - 1 : g.lane;
    int last_lane = 31 - maro_clz(peers);
    int nxt_slot = g.shfl(slot, nxt_lane);
    int last_slot = g.shfl(slot, want ? last_lane : g.lane);
    g.sync();
    if (g.lane == 0) { r.c[C_FREE_TOP] = top - n; r.c[C_Q_COUNT] += n; }
#if defined(MARO_HOST_EMULATION) && defined(MARO_TRACK_QPEAK)  // tools/cim_queue_peak.py: high-water mark of the calendar queue
    if (g.lane == 0 && r.c[C_Q_COUNT] > maro_emul_qpeak) maro_emul_qpeak = r.c[C_Q_COUNT];
#endif
    if (want) {
        int32_t* e = r.q + slot * 2;
        e[0] = w0; e[1] = qty;
        nx[slot] = (uint16_t)(above ? nxt_slot : Q_NIL);
        if (!below) {  // first lane of this bucket's run: splice the run after the current tail
            int32_t* bk = q_bucket(s, r) + b;
            int hb = *bk, tail = (hb >> 16) & 0xffff;
            if (tail == Q_NIL) *bk = slot | (last_slot << 16);
            else { nx[tail] = (uint16_t)slot; *bk = (hb & 0xffff) | (last_slot << 16); }
        }
    }
    g.sync();
}

// ------------------------------------------------------------------------------------------------
// Static-table helpers (maro/data_lib/cim/vessel_*_wrapper.py, vessel_future_stops_prediction.py)
// ------------------------------------------------------------------------------------------------
// Vessel._update_remaining_space (vessel.py:113-120); total_space = floor(capacity / container_volume)
// (kSmall: container volume 1)
template <bool kSmall = false>
MARO_DEV int total_space(const CimShape& s, int cap) { return kSmall || s.vol_is_one ? cap : (int)maro_floor((double)cap / s.vol); }
template <bool kSmall = false>
MARO_DEV void vessel_update_space(const CimShape& s, const Replica& r, int v) {
    VA(s, r, VA_REMAINING_SPACE, v) = total_space<kSmall>(s, VA(s, r, VA_CAPACITY, v)) - VA(s, r, VA_FULL, v) - VA(s, r, VA_EMPTY, v);
}

// VesselPastStopsWrapper.__getitem__ (:23-38) + Vessel.set_stop_list (vessel.py:91-111) — one lane per vessel
MARO_DEV void set_past_stops(const CimShape& s, const Replica& r, int v, int last_loc_idx, int loc_idx) {
    int n = s.past;
    if (n <= 0) return;
    int last_stop_idx = loc_idx + (last_loc_idx == loc_idx ? 0 : -1);
    int start = last_stop_idx - n + 1;
    if (start < 0) start = 0;
    int sb = TBL_I(r, s.t_stop_offset, v);
    int ns = TBL_I(r, s.t_stop_offset, v + 1) - sb;
    int end = loc_idx < ns ? loc_idx : ns;
    int cnt = end - start;
    if (cnt < 0) cnt = 0;
    int pad = n - cnt;
    int32_t* lp = r.f + s.o_past + v * n;
    int32_t* lt = r.f + s.o_past_tick + v * n;
    for (int i = 0; i < n; i++) {
        if (i < pad) { lp[i] = -1; lt[i] = -1; }
        else {
            int si = sb + start + (i - pad);
            lp[i] = TBL_I(r, s.t_stop_port, si);
            lt[i] = TBL_I(r, s.t_stop_arrival, si);
        }
    }
}

// VesselFutureStopsPrediction._predict_future_stops (:49-85), serial form: used by reset (one lane per vessel)
MARO_DEV void predict_serial(const CimShape& s, const Replica& r, int v, int stop_idx, bool lists, bool plans) {
    int rt = TBL_I(r, s.t_vessel_route, v);
    int rbase = TBL_I(r, s.t_route_offset, rt);
    int rl = TBL_I(r, s.t_route_offset, rt + 1) - rbase;
    int lbase = TBL_I(r, s.t_vessel_leg_offset, v);
    int arrival = TBL_I(r, s.t_stop_arrival, TBL_I(r, s.t_stop_offset, v) + stop_idx);
    int loc = (TBL_I(r, s.t_vessel_route_start, v) + stop_idx) % rl;
    int n = rl > s.fut ? rl : s.fut;
    for (int k = 0; k < n; k++) {
        arrival += TBL_I(r, s.t_vessel_leg, lbase + loc);
        loc = loc + 1 == rl ? 0 : loc + 1;
        int port = TBL_I(r, s.t_route_port, rbase + loc);
        if (lists && k < s.fut) { r.f[s.o_fut + v * s.fut + k] = port; r.f[s.o_fut_tick + v * s.fut + k] = arrival; }
        if (plans && k < rl) r.f[s.o_vp + v * s.P + port] = arrival;
    }
}

// ------------------------------------------------------------------------------------------------
// Phase (b): events queued for this tick by earlier ticks.  _on_full_return (:499-522), _on_empty_return (:695-706),
// _on_discharge (:658-693) are pure adds -> shared-memory atomics in any order; RETURN_EMPTY pushes keep lane order.
// ------------------------------------------------------------------------------------------------
template <int G, bool kGeneral, bool kSmall>
MARO_DEV int run_bucket(const CimShape& s, const Grp<G>& g, const Replica& r, int tick) {
    int32_t* bk = q_bucket(s, r) + (tick & (s.QH - 1));
    int head = *bk & 0xffff;
    if (head == Q_NIL) return 0;
    g.sync();
    if (g.lane == 0) *bk = Q_NIL | (Q_NIL << 16);
    int nev = 0;
    uint16_t* fs = q_free(s, r);
    const uint16_t* nx = q_next(s, r);
    while (head != Q_NIL) {  // group-uniform
        // lane i walks to the i-th event of the list (Q_NIL past the end)
        int my = head;
        for (int h = 0; h < g.lane && my != Q_NIL; h++) my = nx[my];
        bool valid = my != Q_NIL;
        int w0 = 0, qty = 0, nxt = Q_NIL;
        if (valid) { w0 = r.q[my * 2]; qty = r.q[my * 2 + 1]; nxt = nx[my]; }
        head = g.shfl(nxt, G - 1);  // continuation for lists longer than G
        uint32_t vb = g.ballot(valid);
        int n = maro_popc(vb);
        int type = w0 & 0xff, a = (w0 >> 8) & 0xff, c = (w0 >> 24) & 0xff, b = (w0 >> 16) & 0xff;
        bool is_dis = valid && type == DE_DISCHARGE_FULL;
        if (valid) {
            if (type == DE_RETURN_FULL) {
                atomic_add(&PA(s, r, PA_ON_SHIPPER, a), -qty);
                atomic_add(&PA(s, r, PA_FULL, a), qty);
                atomic_add(&r.f[s.o_fop + a * s.P + b], qty);
            } else if (type == DE_RETURN_EMPTY) {
                atomic_add(&PA(s, r, PA_ON_CONSIGNEE, a), -qty);
                atomic_add(&PA(s, r, PA_EMPTY, a), qty);
            } else {  // DISCHARGE_FULL: a = vessel, b = from port, c = port
                atomic_add(&VA(s, r, VA_FULL, a), -qty);
                atomic_add(&VA(s, r, VA_REMAINING_SPACE, a), qty);
                atomic_add(&PA(s, r, PA_ON_CONSIGNEE, c), qty);
                atomic_add(&r.f[s.o_fov + a * s.P + c], -qty);
            }
        }
        // empty-return buffer ticks of the discharges (port_buffer_tick_wrapper.py:29-35), drawn in event order
        uint32_t db = g.ballot(is_dis);
        int buf = 0;
        if (db) {
            if (kGeneral && s.buffer_noise) {
                int nd = maro_popc(db);
                int drank = maro_popc(db & ((1u << g.lane) - 1u));
                MtView mv = mt_reserve(s, g, r, 1, 2 * nd);
                if (is_dis) {
                    double u = mt_uniform01(mv.at(2 * drank), mv.at(2 * drank + 1));
                    buf = (int)maro_ceil(noised(TBL_D(r, s.t_erb_d, c), TBL_D(r, s.t_ern_d, c), u));
                }
            } else if (is_dis) {
                buf = TBL_I(r, s.t_erb_i, c);
            }
            bool imm = is_dis && buf == 0;  // immediate RETURN_EMPTY right after the discharge
            if (imm) {
                atomic_add(&PA(s, r, PA_ON_CONSIGNEE, c), -qty);
                atomic_add(&PA(s, r, PA_EMPTY, c), qty);
            }
            nev += maro_popc(g.ballot(imm));
        }
        // recycle this chunk's slots, then append the RETURN_EMPTY events
        g.sync();
        int top = r.c[C_FREE_TOP];
        if (valid) fs[top + g.lane] = (uint16_t)my;
        g.sync();
        if (g.lane == 0) { r.c[C_FREE_TOP] = top + n; r.c[C_Q_COUNT] -= n; }
        g.sync();
        if (db) {
            if (!kGeneral && (kSmall || s.DL)) {
                if (is_dis && buf > 0 && tick + buf < s.max_tick) {
                    int32_t* sl = dl_slot(s, r, tick + buf);
                    atomic_add(&sl[s.P * s.P + c], qty);
                    atomic_add(&sl[s.P * s.P + s.P + 1], 1);
                }
                g.sync();
            } else {
                group_push(s, g, r, is_dis && buf > 0, tick, tick + buf, DE_RETURN_EMPTY | (c << 8), qty);
            }
        }
        nev += n;
    }
    g.sync();
    return nev;
}

// ------------------------------------------------------------------------------------------------
// Phase (c): this tick's ORDER events.  _on_order_generated (:448-497) for up to G orders at a time:
// orders of one source port consume `empty` in sequence -> segmented prefix sum (orders arrive sorted by source).
// `get(i, w, q)` yields order i as {src | dst << 8, qty}.
// ------------------------------------------------------------------------------------------------
template <int G, bool kGeneral, bool kSmall, class Get>
MARO_DEV int run_orders(const CimShape& s, const Grp<G>& g, const Replica& r, int tick, int n_orders, Get get) {
    int nev = 0;
    for (int base = 0; base < n_orders; base += G) {
        int i = base + g.lane;
        bool valid = i < n_orders;
        int w = 0, q = 0;
        if (valid) get(i, w, q);
        int src = valid ? (w & 0xff) : (0x100 + g.lane), dst = (w >> 8) & 0xff;
        int empty0 = valid ? PA(s, r, PA_EMPTY, src) : 0;
        int S = scan_incl_seg(g, q, src);
        int E = S < empty0 ? S : empty0;
        int Ep = (S - q) < empty0 ? (S - q) : empty0;
        int exec = E - Ep;
        int src_next = g.shfl_down(src, 1);
        bool is_last = valid && (g.lane == G - 1 || src_next != src);
        g.sync();
        if (is_last) {  // one lane per source port commits the port's totals
            int booking = PA(s, r, PA_BOOKING, src) + S;
            int shortage = PA(s, r, PA_SHORTAGE, src) + (S - E);
            PA(s, r, PA_BOOKING, src) = booking;
            PA(s, r, PA_ACC_BOOKING, src) += S;
            PA(s, r, PA_SHORTAGE, src) = shortage;
            PA(s, r, PA_ACC_SHORTAGE, src) += S - E;
            PA(s, r, PA_FULFILLMENT, src) = booking - shortage;  // _on_booking_changed / _on_shortage_changed
            PA(s, r, PA_EMPTY, src) = empty0 - E;
            PA(s, r, PA_ON_SHIPPER, src) += E;
        }
        g.sync();
        // full-return buffer ticks, drawn in order (one draw per ORDER)
        int buf = 0;
        int nv = base + G <= n_orders ? G : n_orders - base;
        if (kGeneral && s.buffer_noise) {
            MtView mv = mt_reserve(s, g, r, 1, 2 * nv);
            if (valid) {
                double u = mt_uniform01(mv.at(2 * g.lane), mv.at(2 * g.lane + 1));
                buf = (int)maro_ceil(noised(TBL_D(r, s.t_frb_d, src), TBL_D(r, s.t_frn_d, src), u));
            }
        } else if (valid) {
            buf = TBL_I(r, s.t_frb_i, src);
        }
        bool imm = valid && buf == 0;  // immediate RETURN_FULL (_on_full_return :499-522)
        if (imm) {
            atomic_add(&PA(s, r, PA_ON_SHIPPER, src), -exec);
            atomic_add(&PA(s, r, PA_FULL, src), exec);
            atomic_add(&r.f[s.o_fop + src * s.P + dst], exec);
        }
        nev += nv + maro_popc(g.ballot(imm));
        if (!kGeneral && (kSmall || s.DL)) {
            if (valid && buf > 0 && tick + buf < s.max_tick) {
                int32_t* sl = dl_slot(s, r, tick + buf);
                atomic_add(&sl[src * s.P + dst], exec);
                atomic_add(&sl[s.P * s.P + s.P], 1);
            }
            g.sync();
        } else {
            group_push(s, g, r, valid && buf > 0, tick, tick + buf, DE_RETURN_FULL | (src << 8) | (dst << 16), exec);
        }
    }
    return nev;
}

// Reference form of the order generator (leader lane, float64; kept as the readable statement of the algorithm that
// gen_orders_coop distributes over the lanes): CimSyntheticDataContainer._gen_orders (cim_data_container.py:310-398).
// builtin sum() of floats as CPython >= 3.12 evaluates it (bltinmodule.c builtin_sum_impl: first item + int 0, then
// Neumaier's compensated summation, compensation added at the end) — list_sum_normalize (data_lib/cim/utils.py:44-56).
MARO_DEV double py_sum(const double* x, int n) {
    if (n <= 0) return 0.0;
    double f = 0.0 + x[0], c = 0.0;
    for (int i = 1; i < n; i++) {
        double v = x[i], t = f + v;
        if (fabs(f) >= fabs(v)) c += (f - t) + v; else c += (v - t) + f;
        f = t;
    }
    if (c != 0.0 && isfinite(c)) f += c;
    return f;
}

// Writes {src | dst << 8, qty} pairs to `out` and returns the count.  Scratch doubles live in the MT block.
MARO_DEV int gen_orders_serial(const CimShape& s, const Replica& r, int tick, int total_empty, int32_t* out, double* dscr) {
    int orders_to_gen = TBL_I(r, s.t_order_proportion, tick);
    if (s.order_mode == 1) {
        int delta = s.total_containers - total_empty;
        if (orders_to_gen <= delta) return 0;
        orders_to_gen -= delta;
    }
    int remaining = orders_to_gen, n = 0;
    double* srcd = dscr;
    double* tgtd = dscr + s.P;
    for (int p = 0; p < s.P; p++)
        srcd[p] = s.order_noise ? apply_noise_serial(r, 0, TBL_D(r, s.t_sb_d, p), TBL_D(r, s.t_sn_d, p))
                                : TBL_D(r, s.t_sb_d, p) + 0.0;
    const double tot = py_sum(srcd, s.P);
    for (int p = 0; p < s.P; p++) {
        if (remaining == 0) break;
        int lo = TBL_I(r, s.t_target_offset, p), hi = TBL_I(r, s.t_target_offset, p + 1);
        for (int i = lo; i < hi; i++)
            tgtd[i - lo] = s.order_noise ? apply_noise_serial(r, 0, TBL_D(r, s.t_tb_d, i), TBL_D(r, s.t_tn_d, i))
                                         : TBL_D(r, s.t_tb_d, i) + 0.0;
        const double ttot = py_sum(tgtd, hi - lo);
        double sp = srcd[p];
        if (tot != 0.0) sp = sp / tot;
        int cur = (int)maro_ceil((double)orders_to_gen * sp);
        if (cur > remaining) cur = remaining;
        remaining -= cur;
        if (cur > 0) {
            int trem = cur;
            for (int i = lo; i < hi; i++) {
                double tp = tgtd[i - lo];
                if (ttot != 0.0) tp = tp / ttot;
                int num = (int)maro_ceil((double)cur * tp);
                if (num > trem) num = trem;
                trem -= num;
                if (num > 0) { out[2 * n] = p | (TBL_I(r, s.t_target_port, i) << 8); out[2 * n + 1] = num; n++; }
            }
        }
    }
    return n;
}


// Cooperative noisy order generation: the same arithmetic as gen_orders_serial, spread over the lane group.
// Exactness notes: (i) every python `sum()` stays one sequential float64 chain (py_sum; one lane per chain: the source total
// on the leader, each port's target total on that port's lane); (ii) the running-remainder clamps are integer scans done
// sequentially per chain; (iii) MT19937 draws are addressed by rank: P source draws, then the targets of every port
// before the `remaining == 0` break — those ports are a prefix, so their targets are a prefix of the flattened target
// table and target i is draw P + i.  Scratch layout (global, per replica): srcd[P] | tgtd[T] doubles, then ints.
template <int G>
MARO_DEV int gen_orders_coop(const CimShape& s, const Grp<G>& g, const Replica& r, int tick, int total_empty,
                             int32_t* out, double* dscr) {
    int orders_to_gen = TBL_I(r, s.t_order_proportion, tick);
    if (s.order_mode == 1) {
        int delta = s.total_containers - total_empty;
        if (orders_to_gen <= delta) return 0;
        orders_to_gen -= delta;
    }
    const int P = s.P;
    double* srcd = dscr;
    double* tgtd = dscr + P;
    double* bcast = dscr + P + ((s.max_targets + 1) & ~1);      // one float64 broadcast slot
    int32_t* isc = reinterpret_cast<int32_t*>(bcast + 1);       // ints: cur[P] | c2[T] | cnt[P]
    int32_t* cur = isc;
    int32_t* c2 = isc + P;
    int32_t* cnt = c2 + s.max_targets;
    // ---- 1. noised source shares (draw p = rank p)
    for (int p0 = 0; p0 < P; p0 += G) {
        int nv = P - p0 < G ? P - p0 : G;
        int p = p0 + g.lane;
        if (s.order_noise) {
            MtView mv = mt_reserve(s, g, r, 0, 2 * nv);
            if (p < P) srcd[p] = noised(TBL_D(r, s.t_sb_d, p), TBL_D(r, s.t_sn_d, p), mt_uniform01(mv.at(2 * g.lane), mv.at(2 * g.lane + 1)));
        } else if (p < P) {
            srcd[p] = TBL_D(r, s.t_sb_d, p) + 0.0;
        }
    }
    g.sync();
    // ---- 2. total (left to right) + per-port ceil, then the sequential clamp; `pb` = first port not reached (break)
    if (g.lane == 0) {
        *bcast = py_sum(srcd, P);
    }
    g.sync();
    const double tot = *bcast;
    for (int p0 = 0; p0 < P; p0 += G) {
        int p = p0 + g.lane;
        if (p < P) {
            double sp = srcd[p];
            if (tot != 0.0) sp = sp / tot;
            cur[p] = (int)maro_ceil((double)orders_to_gen * sp);
        }
    }
    g.sync();
    if (g.lane == 0) {
        int remaining = orders_to_gen, pb = P;
        for (int p = 0; p < P; p++) {
            if (remaining == 0) { pb = p; break; }
            int c = cur[p];
            if (c > remaining) c = remaining;
            remaining -= c;
            cur[p] = c;
        }
        r.c[C_N_ORDERS] = pb;
    }
    g.sync();
    const int pb = r.c[C_N_ORDERS];
    const int T = TBL_I(r, s.t_target_offset, pb);  // targets of ports [0, pb) are drawn
    // ---- 3. noised target shares (draw P + i)
    for (int i0 = 0; i0 < T; i0 += G) {
        int nv = T - i0 < G ? T - i0 : G;
        int i = i0 + g.lane;
        if (s.order_noise) {
            MtView mv = mt_reserve(s, g, r, 0, 2 * nv);
            if (i < T) tgtd[i] = noised(TBL_D(r, s.t_tb_d, i), TBL_D(r, s.t_tn_d, i), mt_uniform01(mv.at(2 * g.lane), mv.at(2 * g.lane + 1)));
        } else if (i < T) {
            tgtd[i] = TBL_D(r, s.t_tb_d, i) + 0.0;
        }
    }
    g.sync();
    // ---- 4. one lane per port: target total (left to right), per-target ceil + clamp, order count
    for (int p0 = 0; p0 < pb; p0 += G) {
        int p = p0 + g.lane;
        if (p < pb) {
            int lo = TBL_I(r, s.t_target_offset, p), hi = TBL_I(r, s.t_target_offset, p + 1);
            const double ttot = py_sum(tgtd + lo, hi - lo);
            int c = cur[p], trem = c, n = 0;
            for (int i = lo; i < hi; i++) {
                int num = 0;
                if (c > 0) {
                    double tp = tgtd[i];
                    if (ttot != 0.0) tp = tp / ttot;
                    num = (int)maro_ceil((double)c * tp);
                    if (num > trem) num = trem;
                    trem -= num;
                }
                c2[i] = num;
                n += num > 0;
            }
            cnt[p] = n;
        }
    }
    g.sync();
    // ---- 5. compact the orders in (port, target) order
    int base = 0;
    for (int p0 = 0; p0 < pb; p0 += G) {
        int p = p0 + g.lane;
        int n = p < pb ? cnt[p] : 0;
        int incl = scan_incl(g, n);
        int at = base + incl - n;
        if (p < pb && n > 0) {
            int lo = TBL_I(r, s.t_target_offset, p), hi = TBL_I(r, s.t_target_offset, p + 1);
            for (int i = lo; i < hi; i++)
                if (c2[i] > 0) { out[2 * at] = p | (TBL_I(r, s.t_target_port, i) << 8); out[2 * at + 1] = c2[i]; at++; }
        }
        base += g.shfl(incl, G - 1);
    }
    g.sync();
    return base;
}

// ------------------------------------------------------------------------------------------------
// Phase (d): VESSEL_ARRIVAL (:600-632) + LOAD_FULL (:524-598) of one arriving vessel, lanes over route positions.
// ------------------------------------------------------------------------------------------------
template <int G, bool kGeneral, bool kSmall>
MARO_DEV void run_arrival(const CimShape& s, const Grp<G>& g, const Replica& r, int tick, int v) {
    const int loc = VA(s, r, VA_NEXT_LOC_IDX, v);
    const int sb = TBL_I(r, s.t_stop_offset, v);
    const int ns = TBL_I(r, s.t_stop_offset, v + 1) - sb;
    const int port = TBL_I(r, s.t_stop_port, sb + loc);
    const int rt = TBL_I(r, s.t_vessel_route, v);
    const int rbase = TBL_I(r, s.t_route_offset, rt);
    const int rl = TBL_I(r, s.t_route_offset, rt + 1) - rbase;
    const int lbase = TBL_I(r, s.t_vessel_leg_offset, v);
    // ---- _on_arrival: future stop list + sailing plan = prefix sums of the no-noise legs after this stop
    {
        int pos0 = (TBL_I(r, s.t_vessel_route_start, v) + loc) % rl;
        int arrival0 = TBL_I(r, s.t_stop_arrival, sb + loc);
        int n = rl > s.fut ? rl : s.fut;
        GROUP_CHUNKS(b0, n) {  // n <= G in every shipped topology; loop keeps it general
            int k = b0 + g.lane;
            int pos = pos0 + k;  // pos0 < rl and k < max(rl, fut): a few conditional subtractions instead of a division
            while (pos >= rl) pos -= rl;
            int leg = k < n ? TBL_I(r, s.t_vessel_leg, lbase + pos) : 0;
            int cum = scan_incl(g, leg);
            int arr = arrival0 + cum;
            int nport = TBL_I(r, s.t_route_port, rbase + (pos + 1 == rl ? 0 : pos + 1));
            if (k < s.fut) { r.f[s.o_fut + v * s.fut + k] = nport; r.f[s.o_fut_tick + v * s.fut + k] = arr; }
            // plans: a port that appears twice within one route period keeps the later arrival (dict overwrite order)
            uint32_t same = g.match(k < rl ? nport : (0x1000 + g.lane));
            bool last_of_port = (same >> g.lane) <= 1u;
            if (k < rl && last_of_port) r.f[s.o_vp + v * s.P + nport] = arr;
            arrival0 += g.shfl(cum, G - 1);
        }
    }
    // ---- _on_full_load
    const int cap = VA(s, r, VA_CAPACITY, v);
    int full = VA(s, r, VA_FULL, v);
    int acceptable = kSmall || s.vol_is_one ? cap - full : (int)maro_floor(((double)cap - (double)full * s.vol) / s.vol);
    if (acceptable < 0) acceptable = 0;
    int total_loaded = 0;
    g.sync();
    GROUP_CHUNKS(b0, rl) {  // reachable stops: stops[loc + 1 : loc + 1 + route_len]
        int k = b0 + g.lane;
        int si = loc + 1 + k;
        bool valid = k < rl && si < ns;
        int next_port = valid ? TBL_I(r, s.t_stop_port, sb + si) : 0;
        // a port reachable twice: the first occurrence sees the pending cargo, later ones whatever is left (0 if
        // the first took it all; nothing if acceptable ran out) -> only the first occurrence carries `pending`
        uint32_t same = g.match(valid ? next_port : (0x1000 + g.lane));
        bool first = (same & ((1u << g.lane) - 1u)) == 0;
        int pending = valid && first ? r.f[s.o_fop + port * s.P + next_port] : 0;
        if (pending < 0) pending = 0;
        int A = scan_incl(g, pending);
        int hi = A < acceptable ? A : acceptable;
        int lo = (A - pending) < acceptable ? (A - pending) : acceptable;
        int loaded = hi - lo;
        if (loaded > 0) {
            r.f[s.o_fop + port * s.P + next_port] = pending - loaded;
            r.f[s.o_fov + v * s.P + next_port] += loaded;
        }
        if (!kGeneral && (kSmall || s.due_R)) {  // lanes hold distinct stops: plain adds; the drop rules of group_push
            if (loaded > 0 && TBL_I(r, s.t_stop_arrival, sb + si) < s.max_tick) {
                int32_t* sl = due_slot(s, r, v, si);
                sl[0] += loaded;
                sl[1] += 1;
            }
            if (!kSmall) g.sync();  // (a later chunk may read the pending cargo this one wrote)
        } else {
            group_push(s, g, r, loaded > 0, tick, valid ? TBL_I(r, s.t_stop_arrival, sb + si) : 0,
                       DE_DISCHARGE_FULL | (v << 8) | (port << 16) | (next_port << 24), loaded);
        }
        int chunk = g.shfl(hi, G - 1);
        total_loaded += chunk;
        acceptable -= chunk;
    }
    if (g.lane == 0) {
        VA(s, r, VA_LAST_LOC_IDX, v) = loc;
        VA(s, r, VA_IS_PARKING, v) = 1;
        VA(s, r, VA_LOC_PORT_IDX, v) = port;
        PA(s, r, PA_FULL, port) -= total_loaded;
        full += total_loaded;
        VA(s, r, VA_FULL, v) = full;
        int empty = VA(s, r, VA_EMPTY, v);
        int total_container = full + empty;
        int early = 0;
        const bool vol1 = kSmall || s.vol_is_one;
        bool over = vol1 ? total_container > cap : (double)total_container * s.vol > (double)cap;
        if (over) {
            early = total_container - (vol1 ? cap : (int)maro_ceil((double)cap / s.vol));
            empty -= early;
            VA(s, r, VA_EMPTY, v) = empty;
            PA(s, r, PA_EMPTY, port) += early;
        }
        VA(s, r, VA_EARLY_DISCHARGE, v) = early;
        VA(s, r, VA_REMAINING_SPACE, v) = total_space<kSmall>(s, cap) - full - empty;
    }
    g.sync();
}

// _on_departure (:634-656) — one lane per vessel
MARO_DEV void on_departure(const CimShape& s, const Replica& r, int v) {
    int next = VA(s, r, VA_NEXT_LOC_IDX, v) + 1;
    VA(s, r, VA_NEXT_LOC_IDX, v) = next;
    VA(s, r, VA_IS_PARKING, v) = 0;
    VA(s, r, VA_LOC_PORT_IDX, v) = -1;
    set_past_stops(s, r, v, VA(s, r, VA_LAST_LOC_IDX, v), next);
}

struct Act4 { int32_t v, p, qty, type; };

template <bool kSmall = false>
MARO_DEV int frame_index_of(const CimShape& s, int tick) {
    return kSmall || s.res_is_one ? tick - s.start_tick : (tick - s.start_tick) / s.resolution;
}

// _on_action_received (:708-748).  Lane k holds action k (loaded with one 128-bit read); the leader lane applies them in
// order.  Returns false where the reference would raise AssertionError.
template <int G, bool kSmall>
MARO_DEV bool on_actions(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k, const Act4& mine, int n) {
    bool ok = true;
    for (int i = 0; i < n; i++) {
        int v = g.shfl(mine.v, i), p = g.shfl(mine.p, i), move = g.shfl(mine.qty, i), type = g.shfl(mine.type, i);
        if (g.lane != 0 || !ok) continue;
        if (type == 2) continue;  // Joint mode: `None` for this decision event (an empty action list, core.py:308-309)
        if (v < 0 || v >= s.V || p < 0 || p >= s.P || move < 0) { ok = false; continue; }
        int port_empty = PA(s, r, PA_EMPTY, p), vessel_empty = VA(s, r, VA_EMPTY, v);
        if (type == 1) {  // DISCHARGE
            if (!(move <= vessel_empty)) { ok = false; continue; }
            PA(s, r, PA_EMPTY, p) = port_empty + move;
            VA(s, r, VA_EMPTY, v) = vessel_empty - move;
        } else {
            int space = VA(s, r, VA_REMAINING_SPACE, v);
            if (!(move <= (port_empty < space ? port_empty : space))) { ok = false; continue; }
            PA(s, r, PA_EMPTY, p) = port_empty - move;
            VA(s, r, VA_EMPTY, v) = vessel_empty + move;
        }
        vessel_update_space<kSmall>(s, r, v);
        k.opnum += move;  // (leader lane)
        // port.transfer_cost (float32 attr) += move: python float (double) add, stored back as float32
        float tc = maro_i2f(PA(s, r, PA_TRANSFER_COST, p));
        PA(s, r, PA_TRANSFER_COST, p) = maro_f2i(maro_d2f((double)tc + (double)move));
        r.f[s.o_vp + v * s.P + p] += TBL_I(r, s.t_vessel_period, v);
    }
    return ok;
}

// ------------------------------------------------------------------------------------------------
// Snapshot: copy the live frame into ring row (frame_index % ring_rows)
// (FrameBase.take_snapshot -> NPSnapshotList.take_snapshot, np_backend.pyx:481-518).
// On the device the row leaves shared memory as ONE TMA bulk store (cp.async.bulk shared -> global) issued by the leader
// lane; snapshot_wait() must run before the frame is modified again (the engine has then read the source: ~200 cycles
// for a 900-byte row, measured with tools/microbench/tma_s2g_latency.cu, against ~850 for an 8-lane 128-bit copy loop).
// ------------------------------------------------------------------------------------------------
#ifndef MARO_HOST_EMULATION
__device__ __forceinline__ void snapshot_wait_lane() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all bulk stores of this thread have been written (not merely read): once, before the kernel ends (the full wait
// compiles to DEPBAR + CCTL.IVALL, an L1 invalidation — far too expensive per snapshot)
__device__ __forceinline__ void snapshot_drain_lane() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
#endif
template <int G>
MARO_DEV void snapshot_wait(const Grp<G>& g) {
#ifndef MARO_HOST_EMULATION
    if (g.lane == 0) snapshot_wait_lane();
#endif
    g.sync();
}

// the copy of the frame into its ring row (take_snapshot without the counters)
template <int G>
MARO_DEV void snapshot_store(const CimShape& s, const Grp<G>& g, const Replica& r, int frame_index) {
    int row = frame_index < s.ring_rows ? frame_index : frame_index % s.ring_rows;
    int32_t* dst = r.snap + (int64_t)row * s.FWp;
#ifdef MARO_HOST_EMULATION
    g.sync();
    LANE_LOOP(i, s.FWp) dst[i] = r.f[i];
#else
    // every lane's generic-proxy writes to the frame become visible to the async proxy, then the leader issues the copy.
    // Bulk stores of one thread are carried out in issue order (tools/microbench/tma_s2g_cold.cu: 2.4 M back-to-back pairs
    // to one row, never reordered), so the several snapshots of a decision tick (they share a ring row) need no full
    // wait_group between them — which would cost a CCTL.IVALL (L1 invalidation) each time.
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    g.sync();
    if (g.lane == 0) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"((uint32_t)__cvta_generic_to_shared(r.f)),
                     "r"((uint32_t)s.FWp * 4u)
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
#endif
    if (g.lane == 0) r.snap_frame[row] = frame_index;
}

template <int G>
MARO_DEV void take_snapshot(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k, int frame_index) {
    snapshot_store(s, g, r, frame_index);
    k.last_frame = frame_index;
    k.nsnaps += 1;
    k.snap_pending = false;  // (a pending pre-decision snapshot is always of this frame index: same row, now overwritten)
}

// Fused rollouts (replica_step<..., kDeferSnap = true>) take the pre-decision snapshot only logically: inside a launch its ring
// row is always overwritten before anything can read it -- the decision's tick ends with the snapshot of the same frame index
// (same row), and between the two only the device agent runs, which reads the decision row, never the ring.  The row becomes
// observable only if the launch (or slice) ends while the replica waits on that decision; then the frame is still exactly the
// pre-decision frame (nothing modifies it after the decision), and this writes it.  Call once per work item before the write-back.
template <int G, bool kSmall>
MARO_DEV void flush_deferred_snapshot(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k) {
    if (!k.snap_pending) return;  // (group-uniform)
    snapshot_store(s, g, r, frame_index_of<kSmall>(s, k.tick));
    k.snap_pending = false;
}

// Output rows are written with 128-bit / 64-bit stores (they may live in mapped host memory: one PCIe write each).
MARO_DEV void store_out(int32_t* dec, int64_t* met, const int32_t* od, int64_t m0, int64_t m1, int64_t m2) {
#ifdef MARO_HOST_EMULATION
    for (int i = 0; i < 8; i++) dec[i] = od[i];
#else
    reinterpret_cast<int4*>(dec)[0] = make_int4(od[0], od[1], od[2], od[3]);
    reinterpret_cast<int4*>(dec)[1] = make_int4(od[4], od[5], od[6], od[7]);
#endif
    met[0] = m0; met[1] = m1; met[2] = m2;
}

// ------------------------------------------------------------------------------------------------
// One Env.step for one replica.  `act`/`n_act` are this replica's action rows; `dec` (8 int32) and `met`
// (3 int64) its output rows.  All lanes of the group call this together.
// ------------------------------------------------------------------------------------------------
// kGeneral = false compiles the noise-free fast path only (static order schedule, integer buffer ticks, no MT19937).
// kSmall (with kGeneral = false) compiles the small-topology path: resolution 1, container volume 1, Sequential mode, delay
// lines on, and P, V, route lengths and fut <= G (cim_small_ok) -- every lane loop over them is one pass, the vessel cursors
// live in Ctl.  Sizes and table offsets stay runtime values.
// The control state is `k` (ctl_load before, ctl_store after: the control block in shared memory is stale in between).
// kDeferSnap (fused rollouts only): the pre-decision snapshot is left pending in `k` (flush_deferred_snapshot).
template <int G, bool kGeneral, bool kSmall = false, bool kDeferSnap = false>
MARO_DEV void replica_step(const CimShape& s, const Grp<G>& g, const Replica& r, Ctl& k, const Act4& act, int n_act,
                           int32_t* dec, int64_t* met) {
    static_assert(!(kGeneral && kSmall), "the small-topology path is noise-free");
    const bool joint = !kSmall && s.joint;
    const bool res1 = kSmall || s.res_is_one;
    const bool due = !kGeneral && (kSmall || s.due_R);  // discharges on the due rings instead of the calendar queue
    int state = k.state;
    int nev = 0;
    if (state >= ST_DONE) {  // StopIteration -> (None, None, True)   core.py:128-131
        g.sync();
        if (state == ST_DONE) k.state = ST_FINISHED;
        if (g.lane == 0) {
            int32_t od[8] = {0, 0, 0, 0, 0, 0, 2, 0};
            store_out(dec, met, od, 0, 0, 0);
        }
        g.sync();
        return;
    }
    if (state == ST_AWAIT) {
        // _assign_action (core.py:301-315): the decision event finishes, TAKE_ACTION runs as its immediate event
        g.sync();
        int n_apply = n_act;
        if (joint) {  // answer k belongs to the k-th decision of the tick; surplus answers are dropped (zip, core.py:362)
            const uint64_t pend = k.arr;
            int n_dec = 0;
            for (uint64_t m = pend; m; m &= m - 1) n_dec++;
            n_apply = n_act < n_dec ? n_act : n_dec;
        }
        const bool ok = g.ballot(!on_actions<G, kSmall>(s, g, r, k, act, n_apply)) == 0;  // (decided by the leader lane)
        k.nsteps += 1;
        if (!ok) {
            k.state = ST_ERROR;
            if (g.lane == 0) r.c[C_ERR] = -1;
        }
        g.sync();
        nev += joint ? 2 * n_apply : 2;  // decision event + TAKE_ACTION per answered decision
        if (!ok) {
            if (g.lane == 0) { int32_t od[8] = {0, 0, 0, 0, 0, 0, -1, 0}; store_out(dec, met, od, 0, 0, 0); }
            g.sync();
            return;
        }
        state = ST_DECISIONS;
    } else {
        k.nsteps += 1;
        if (state == ST_START) state = ST_TICK_BEGIN;
    }
    PHASE_MARK(r, PH_ACTIONS);

    int tick = k.tick;
    uint64_t arr = k.arr;
    int dec_pos = k.dec_pos;
    int status = 0, nticks = 0;
    int32_t od[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (;;) {
        if (state == ST_TICK_BEGIN) {
            nticks++;
            // ---- BusinessEngine.step(tick), arrival part (business_engine.py:145-199) + (a) the departures
            // pre-inserted at init (:371-379): one lane per vessel.  The tick of each vessel's next arrival /
            // departure is cached in the control block (updated when they fire), so an idle tick costs two
            // shared-memory compares per vessel and no table walk.  Arrivals are tested on the state at tick start
            // (before this tick's departures), like step().
            int total_empty = 0;
            int ndep = 0;
            arr = 0;
            GROUP_CHUNKS(b0, s.V) {
                const int v = b0 + g.lane;
                const bool in = v < s.V;
                // the vessel's cursors: dep_cursor (C_FIXED + v), next departure tick (+ V), next arrival tick (+ 2V)
                int* cur = kSmall ? nullptr : r.c + C_FIXED + v;
                const bool arrives = in && (kSmall ? k.next_arr : cur[2 * s.V]) == tick;
                if (arrives) {
                    int si = TBL_I(r, s.t_stop_offset, v) + VA(s, r, VA_NEXT_LOC_IDX, v);
                    r.f[s.o_vp + v * s.P + TBL_I(r, s.t_stop_port, si)] = tick;
                    if (kSmall) k.next_arr = NO_TICK; else cur[2 * s.V] = NO_TICK;
                }
                if (kGeneral && s.order_mode == 1 && in) total_empty += VA(s, r, VA_EMPTY, v);
                const bool departs = in && (kSmall ? k.next_dep : cur[s.V]) == tick;
                if (departs) {
                    on_departure(s, r, v);
                    const int dc = (kSmall ? k.dep_cursor : cur[0]) + 1;
                    int sb = TBL_I(r, s.t_stop_offset, v), ns = TBL_I(r, s.t_stop_offset, v + 1) - sb;
                    const int nd = dc < ns ? TBL_I(r, s.t_stop_leave, sb + dc) : NO_TICK;
                    int nl = VA(s, r, VA_NEXT_LOC_IDX, v);
                    const int na = nl < ns ? TBL_I(r, s.t_stop_arrival, sb + nl) : NO_TICK;
                    if (kSmall) { k.dep_cursor = dc; k.next_dep = nd; k.next_arr = na; }
                    else { cur[0] = dc; cur[s.V] = nd; cur[2 * s.V] = na; }
                }
                // (b) for the due rings: the discharges due at this stop (fields disjoint from the departure's)
                if (due && in && (kSmall ? k.due_tick : cur[4 * s.V]) == tick) {
                    const int stop = kSmall ? k.due_stop : cur[3 * s.V];
                    k.ndue += drain_due_stop(s, r, v, stop, tick);
                    const int sb = TBL_I(r, s.t_stop_offset, v), ns = TBL_I(r, s.t_stop_offset, v + 1) - sb;
                    const int nt = stop + 1 < ns ? TBL_I(r, s.t_stop_arrival, sb + stop + 1) : NO_TICK;
                    if (kSmall) { k.due_stop = stop + 1; k.due_tick = nt; }
                    else { cur[3 * s.V] = stop + 1; cur[4 * s.V] = nt; }
                }
                arr |= (uint64_t)g.ballot(arrives) << b0;
                ndep += maro_popc(g.ballot(departs));
            }
            if (kGeneral && s.order_mode == 1) {
                LANE_LOOP(p, s.P) total_empty += PA(s, r, PA_EMPTY, p);
                total_empty = g.sum(total_empty);
            }
            nev += ndep;
            g.sync();
            PHASE_MARK(r, PH_VESSELS);
            // ---- (b) events queued by earlier ticks
            if (!due) nev += run_bucket<G, kGeneral, kSmall>(s, g, r, tick);
            PHASE_MARK(r, PH_BUCKET);
            if (!kGeneral && (kSmall || s.DL)) nev += run_delay_line<G, kSmall>(s, g, r, tick);
            PHASE_MARK(r, PH_DELAY);
            // ---- (c) this tick's orders
            if (!kGeneral || s.order_table) {
                int slot = TBL_I(r, s.t_ord_slot, tick);
                int lo = TBL_I(r, s.t_ord_off, slot), hi = TBL_I(r, s.t_ord_off, slot + 1);
                const int32_t* list = r.t + s.t_ord_list + 2 * lo;
                nev += run_orders<G, kGeneral, kSmall>(s, g, r, tick, hi - lo, [&](int i, int& w, int& q) { w = list[2 * i]; q = list[2 * i + 1]; });
            } else {
                // float64 generation on the leader lane into the replica's scratch area, then cooperative execution
                int32_t* olist = reinterpret_cast<int32_t*>(r.mt + s.mt_scratch + 64);
                double* dscr = reinterpret_cast<double*>(olist + 2 * ((s.max_targets + 1) & ~1));
                g.sync();
                int n = gen_orders_coop(s, g, r, tick, total_empty, olist, dscr);
                nev += run_orders<G, kGeneral, kSmall>(s, g, r, tick, n, [&](int i, int& w, int& q) { w = olist[2 * i]; q = olist[2 * i + 1]; });
            }
            g.sync();
            PHASE_MARK(r, PH_ORDERS);
            // ---- (d) VESSEL_ARRIVAL + LOAD_FULL per arriving vessel, vessel order
            uint64_t m = arr;
            while (m) {
                int v = maro_ffs64(m) - 1;
                m &= m - 1;
                run_arrival<G, kGeneral, kSmall>(s, g, r, tick, v);
                nev += 2;
            }
            PHASE_MARK(r, PH_ARRIVALS);
            dec_pos = 0;
            state = ST_DECISIONS;
        }
        // ---- (e) decision events, one per arriving vessel, vessel order (Sequential mode, core.py:348-353)
        uint64_t m = dec_pos >= 64 ? 0 : (arr >> dec_pos) << dec_pos;
        if (m) {
            int v = maro_ffs64(m) - 1;
            if (kDeferSnap) {  // core.py:345, written by flush_deferred_snapshot if it is ever observable
                k.last_frame = frame_index_of<kSmall>(s, tick);
                k.nsnaps += 1;
                k.snap_pending = true;
            } else {
                take_snapshot(s, g, r, k, frame_index_of<kSmall>(s, tick));  // core.py:345
            }
            if (g.lane == 0) {
                int port = VA(s, r, VA_LOC_PORT_IDX, v);
                int pe = PA(s, r, PA_EMPTY, port), sp = VA(s, r, VA_REMAINING_SPACE, v);
                od[0] = tick; od[1] = port; od[2] = v;
                od[3] = pe < sp ? pe : sp;
                od[4] = VA(s, r, VA_EMPTY, v);
                od[5] = VA(s, r, VA_EARLY_DISCHARGE, v);
                if (joint) {  // rows 1.. : the tick's other decisions, scopes from the same (pre-action) state; then a terminator
                    int n = 1;
                    for (uint64_t rest = m & (m - 1); rest; rest &= rest - 1, n++) {
                        const int v2 = maro_ffs64(rest) - 1, port2 = VA(s, r, VA_LOC_PORT_IDX, v2);
                        const int pe2 = PA(s, r, PA_EMPTY, port2), sp2 = VA(s, r, VA_REMAINING_SPACE, v2);
                        int32_t row[8] = {tick, port2, v2, pe2 < sp2 ? pe2 : sp2, VA(s, r, VA_EMPTY, v2), VA(s, r, VA_EARLY_DISCHARGE, v2),
                                          0, k.ep_step};
                        for (int i = 0; i < 8; i++) dec[8 * n + i] = row[i];
                    }
                    if (n < s.V) dec[8 * n + 6] = 3;  // MARO_STATUS_INACTIVE: end of this step's decision list
                }
            }
            dec_pos = joint ? 64 : v + 1;
            state = ST_AWAIT;
            status = 0;
            PHASE_MARK(r, PH_DECISION);
            break;
        }
        // ---- post_step (business_engine.py:201-224)
        if (res1 || (tick + 1) % s.resolution == 0) {
            g.sync();
            LANE_DIM(p, s.P) PA(s, r, PA_ACC_FULFILLMENT, p) = PA(s, r, PA_ACC_BOOKING, p) - PA(s, r, PA_ACC_SHORTAGE, p);
            take_snapshot(s, g, r, k, frame_index_of<kSmall>(s, tick));
            snapshot_wait(g);  // the row has left the frame: the per-tick resets may overwrite it
            LANE_DIM(p, s.P) {
                PA(s, r, PA_SHORTAGE, p) = 0;
                PA(s, r, PA_BOOKING, p) = 0;
                PA(s, r, PA_FULFILLMENT, p) = 0;
                PA(s, r, PA_TRANSFER_COST, p) = 0;
            }
            g.sync();
        }
        if (tick + 1 == s.max_tick) {
            if (!res1 && (tick + 1) % s.resolution != 0) { take_snapshot(s, g, r, k, frame_index_of(s, tick)); snapshot_wait(g); }  // core.py:376-378
            state = ST_DONE;
            status = 1;
            od[0] = tick;
            PHASE_MARK(r, PH_POST);
            break;
        }
        tick += 1;
        state = ST_TICK_BEGIN;
        PHASE_MARK(r, PH_POST);
    }
    // ---- metrics (business_engine.py:270-282) + control write-back
    g.sync();
    int64_t bk = 0, sh = 0;
    if (s.P <= 8) {  // few ports: the leader adds them up itself (cheaper than two 64-bit shuffle reductions)
        if (g.lane == 0)
            for (int p = 0; p < s.P; p++) { bk += PA(s, r, PA_ACC_BOOKING, p); sh += PA(s, r, PA_ACC_SHORTAGE, p); }
    } else {
        LANE_LOOP(p, s.P) { bk += PA(s, r, PA_ACC_BOOKING, p); sh += PA(s, r, PA_ACC_SHORTAGE, p); }
        bk = g.sum64(bk);
        sh = g.sum64(sh);
    }
    if (r.c[C_ERR] == -2) { state = ST_ERROR; status = -2; }
    k.state = state;
    k.tick = tick;
    k.arr = arr;
    k.dec_pos = dec_pos;
    k.nevents += nev;
    k.nticks += nticks;
    od[6] = status;
    od[7] = k.ep_step;  // ordinal of this env-step inside the episode (0 = first decision)
    k.ep_step += 1;
    if (g.lane == 0) store_out(dec, met, od, bk, sh, k.opnum);
    if (kDeferSnap) g.sync();  // (no bulk read of the frame outstanding: the end-of-tick snapshots wait for theirs)
    else snapshot_wait(g);     // the pre-decision snapshot (if any) has been read: the caller may touch the frame again
    PHASE_COUNT(r, PH_TICKS, nticks);
    PHASE_MARK(r, PH_STORE);
}

// One step on the control block as it stands in memory (ctl_load, replica_step, ctl_store): the form for callers that do
// not keep the control state in registers between steps.
template <int G, bool kGeneral>
MARO_DEV void replica_step(const CimShape& s, const Grp<G>& g, const Replica& r, const Act4& act, int n_act, int32_t* dec,
                           int64_t* met) {
    Ctl k;
    ctl_load<G, false>(s, g, r, k);
    replica_step<G, kGeneral, false>(s, g, r, k, act, n_act, dec, met);
    ctl_store<G, false>(s, g, r, k);
}

// ------------------------------------------------------------------------------------------------
// Env.reset / initial state of one replica (core.py:143-170; business_engine.py:226-242, 314-356, 381-398).
// ------------------------------------------------------------------------------------------------
template <int G>
MARO_DEV void replica_reset(const CimShape& s, const Grp<G>& g, const Replica& r) {
    LANE_LOOP(i, s.FWp) r.f[i] = 0;
    LANE_LOOP(i, s.CWp) if (i < C_NSTEPS_LO || i > C_NSNAPS_HI) r.c[i] = 0;  // cumulative work counters survive
    g.sync();
    LANE_LOOP(p, s.P) {
        PA(s, r, PA_CAPACITY, p) = TBL_I(r, s.t_port_capacity, p);
        PA(s, r, PA_EMPTY, p) = TBL_I(r, s.t_port_init_empty, p);
    }
    LANE_LOOP(i, s.V * s.P) r.f[s.o_vp + i] = -1;
    g.sync();
    LANE_LOOP(v, s.V) {
        VA(s, r, VA_CAPACITY, v) = TBL_I(r, s.t_vessel_capacity, v);
        VA(s, r, VA_ROUTE_IDX, v) = TBL_I(r, s.t_vessel_route, v);
        VA(s, r, VA_EMPTY, v) = TBL_I(r, s.t_vessel_init_empty, v);
        vessel_update_space(s, r, v);
        // _init_vessel_plans
        VA(s, r, VA_IS_PARKING, v) = 1;
        VA(s, r, VA_LOC_PORT_IDX, v) = TBL_I(r, s.t_stop_port, TBL_I(r, s.t_stop_offset, v));
        set_past_stops(s, r, v, 0, 0);
        predict_serial(s, r, v, 0, true, true);
        // departures whose leave tick precedes start_tick are never executed
        int sb = TBL_I(r, s.t_stop_offset, v), ns = TBL_I(r, s.t_stop_offset, v + 1) - sb;
        int dc = 0;
        while (dc < ns && TBL_I(r, s.t_stop_leave, sb + dc) < s.start_tick) dc++;
        r.c[C_FIXED + v] = dc;
        r.c[C_FIXED + s.V + v] = dc < ns ? TBL_I(r, s.t_stop_leave, sb + dc) : NO_TICK;
        r.c[C_FIXED + 2 * s.V + v] = NO_TICK;  // next_loc_idx == 0: no arrival until the first departure
        if (s.due_R) {  // due rings: the first stop due at or after start_tick (nothing is outstanding before it)
            int ds = 0;
            while (ds < ns && TBL_I(r, s.t_stop_arrival, sb + ds) < s.start_tick) ds++;
            r.c[C_FIXED + 3 * s.V + v] = ds;
            r.c[C_FIXED + 4 * s.V + v] = ds < ns ? TBL_I(r, s.t_stop_arrival, sb + ds) : NO_TICK;
        }
    }
    LANE_LOOP(i, 2 * s.V * s.due_R) r.f[s.o_due + i] = 0;
    // queue: all slots on the free stack (slot 0 on top so that allocation order is ascending), empty buckets
    uint16_t* fs = q_free(s, r);
    uint16_t* nx = q_next(s, r);
    LANE_LOOP(i, s.QN) {
        r.q[i * 2 + 0] = 0; r.q[i * 2 + 1] = 0;
        nx[i] = Q_NIL;
        fs[i] = (uint16_t)(s.QN - 1 - i);
    }
    LANE_LOOP(i, s.QH) q_bucket(s, r)[i] = Q_NIL | (Q_NIL << 16);
    LANE_LOOP(i, s.DL * s.dl_stride) r.f[s.o_dl + i] = 0;
    LANE_LOOP(i, s.ring_rows) r.snap_frame[i] = -1;
    if (r.mt) {
        LANE_LOOP(i, 624) {
            r.mt[i] = (uint32_t)TBL_I(r, s.t_mt_order, i);
            r.mt[640 + i] = (uint32_t)TBL_I(r, s.t_mt_buffer, i);
        }
    }
    g.sync();
    if (g.lane == 0) {
        r.c[C_STATE] = ST_START;
        r.c[C_TICK] = s.start_tick;
        r.c[C_FREE_TOP] = s.QN;
        r.c[C_MT_ORDER_IDX] = 624;
        r.c[C_MT_BUFFER_IDX] = 624;
        r.c[C_LAST_FRAME] = -1;
    }
    g.sync();
}

}  // namespace maro
