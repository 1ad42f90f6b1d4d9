// env_common.cuh — pieces shared by the three scenario translation units (cim_env.cu, bike_env.cu, vm_env.cu):
// PTX helpers (mbarrier + TMA bulk copy), the snapshot-query kernel, the handle base class with its device buffers /
// host staging, and the scenario-independent C-ABI helpers.  Everything here has internal or inline linkage.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/maro_b200.h"
#include "cim_core.cuh"  // lane-group primitives
#include "cim_host.hpp"

using namespace maro;

// =====================================================================================================
// PTX helpers: mbarrier + TMA bulk copy (1-D cp.async.bulk)
// =====================================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }


struct QueryArgs {
    const int32_t* snap;
    const int32_t* snap_frame;
    const int32_t* replicas;  // [nr]
    const int32_t* frames;    // [nf]
    const int32_t* nodes;     // [nn]
    const int32_t* attr_off;  // [na] frame word offset of attr (node 0, slot 0)
    const int32_t* attr_slots;
    const int32_t* attr_isf;
    const int32_t* attr_prefix;  // [na] prefix sum of slots
    int nr, nf, nn, na, slots_per_node, ring_rows, FWp;
    int layout, max_slots;  // layout 1 (dynamic backend): [frame][node][attr][max_slots], NaN padding, float32-rounded values
    double* out;
};

// Static layout (np_backend.pyx:536-549): out[rep][frame][node][attr][slot], frames not held by the ring -> 0.
// Dynamic layout (the RawBackend's query, raw/snapshotlist.cpp:244-318 + _raw_backend_.pyx:263-315): every attribute
// padded to `max_slots` slots, result pre-filled with NaN (missing slots, unknown frames), values pass through float32.
static __global__ void cim_query_kernel(const __grid_constant__ QueryArgs q) {
    const int64_t per_rep = (int64_t)q.nf * q.nn * q.slots_per_node;
    const int64_t total = per_rep * q.nr;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t x = i;
        int sl = (int)(x % q.slots_per_node); x /= q.slots_per_node;
        int nd = (int)(x % q.nn); x /= q.nn;
        int fi = (int)(x % q.nf); x /= q.nf;
        int rp = q.replicas[(int)x];
        int ai = 0, slot;
        if (q.layout == 1) {
            ai = sl / q.max_slots;
            slot = sl - ai * q.max_slots;
        } else {
            while (ai + 1 < q.na && q.attr_prefix[ai + 1] <= sl) ai++;
            slot = sl - q.attr_prefix[ai];
        }
        int frame = q.frames[fi];
        double v = q.layout == 1 ? __longlong_as_double(0x7ff8000000000000ll) : 0.0;
        if (q.layout == 1 && slot >= q.attr_slots[ai]) {
            // NaN padding
        } else if (frame >= 0) {
            int row = frame % q.ring_rows;
            if (q.snap_frame[(int64_t)rp * q.ring_rows + row] == frame) {
                int w = q.snap[((int64_t)rp * q.ring_rows + row) * q.FWp + q.attr_off[ai] + q.nodes[nd] * q.attr_slots[ai] + slot];
                v = q.attr_isf[ai] ? (double)__int_as_float(w) : (q.layout == 1 ? (double)(float)w : (double)w);
            }
        }
        q.out[i] = v;
    }
}

// =====================================================================================================
// Host side
// =====================================================================================================
inline thread_local std::string g_err;  // one instance for the library: maro_last_error() lives in cim_env.cu
inline std::mutex g_err_mu;             // + the most recent error of ANY thread (host loops that drive a handle from worker
inline std::string g_err_any;           //   threads report through the thread that joins them)
static int fail(const std::string& m) {
    g_err = m;
    std::lock_guard<std::mutex> lock(g_err_mu);
    g_err_any = m;
    return 1;
}
#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) return fail(std::string(#call) + ": " + cudaGetErrorString(e__));     \
    } while (0)

struct AttrInfo { const char* name; int off, slots, isf, n_nodes; };

// State shared by every scenario handle: device buffers of the replica blocks + snapshot ring, host-call staging,
// query scratch, attribute registry.
struct EnvCommon {
    int device = 0, B = 0;
    int n_sm = 1;  // SMs of the device (grid size of the grid-stride kernels)
    int ring_rows = 0, FW = 0, FWp = 0, SW = 0;
    int off_tick = 0, off_counters = 0;  // word offsets inside a replica's state block
    int dec_words = 8, max_actions = 1, met_words = 3;  // decision row int32 words, metrics row int64 words
    cudaStream_t own_stream = nullptr, stream = nullptr;
    int32_t *d_state = nullptr, *d_snap = nullptr, *d_snap_frame = nullptr;
    // host-call staging
    uint8_t* d_in = nullptr;   // [actions B*A*4 i32][n_actions B i32][active B u8]
    uint8_t* d_out = nullptr;  // [decisions B*dec_words i32][metrics B*3 i64]
    uint8_t *h_in = nullptr, *h_out = nullptr;    // pinned mirrors (mapped into the device address space)
    uint8_t *hd_in = nullptr, *hd_out = nullptr;  // device aliases of h_in / h_out for the zero-copy path
    bool zero_copy = false;
    size_t in_bytes = 0, out_bytes = 0;
    int32_t* d_qidx = nullptr;  // query index scratch
    size_t qidx_cap = 0;
    double* d_qout = nullptr;
    size_t qout_cap = 0;
    std::vector<AttrInfo> attrs[6];
    int n_node_types = 3;
    int query_layout = 0;  // MARO_QUERY_LAYOUT_STATIC / _DYNAMIC (maro_*_set_query_layout)
    // device buffers beyond [state | ring] that belong to the simulation state (RNG streams, topology tables ...): the
    // scenario registers them at create time so that a checkpoint carries them (common_save / common_load)
    struct ExtraBuffer { const char* name; void** d_ptr; size_t bytes; };
    std::vector<ExtraBuffer> ckpt_extra;
    int scenario_id = 0;
};

static void common_free(EnvCommon* e) {
    cudaFree(e->d_state); cudaFree(e->d_snap); cudaFree(e->d_snap_frame);
    cudaFree(e->d_in); cudaFree(e->d_out); cudaFree(e->d_qidx); cudaFree(e->d_qout);
    if (e->h_in) cudaFreeHost(e->h_in);
    if (e->h_out) cudaFreeHost(e->h_out);
    if (e->own_stream) cudaStreamDestroy(e->own_stream);
}

// stream + replica blocks + snapshot ring + host staging (sizes from B / SW / ring_rows / FWp / dec_words / max_actions)
static int common_alloc(EnvCommon* e) {
    CK(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    e->stream = e->own_stream;
    CK(cudaDeviceGetAttribute(&e->n_sm, cudaDevAttrMultiProcessorCount, e->device));
    const size_t B = (size_t)e->B;
    CK(cudaMalloc(&e->d_state, B * e->SW * 4));
    CK(cudaMalloc(&e->d_snap, B * e->ring_rows * e->FWp * 4));
    CK(cudaMalloc(&e->d_snap_frame, B * e->ring_rows * 4));
    // cudaMalloc may hand back memory a freed handle of this process used.  The work counters of the state blocks persist
    // across resets (no reset writes them), so the blocks start from zeros; the ring starts empty.
    CK(cudaMemset(e->d_state, 0, B * e->SW * 4));
    CK(cudaMemset(e->d_snap, 0, B * e->ring_rows * e->FWp * 4));
    CK(cudaMemset(e->d_snap_frame, 0xff, B * e->ring_rows * 4));
    e->in_bytes = B * e->max_actions * 16 + B * 4 + round_up(e->B, 16);
    e->out_bytes = B * e->dec_words * 4 + B * e->met_words * 8;
    CK(cudaMalloc(&e->d_in, e->in_bytes));
    CK(cudaMalloc(&e->d_out, e->out_bytes));
    CK(cudaHostAlloc(&e->h_in, e->in_bytes, cudaHostAllocMapped));
    CK(cudaHostAlloc(&e->h_out, e->out_bytes, cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer((void**)&e->hd_in, e->h_in, 0));
    CK(cudaHostGetDevicePointer((void**)&e->hd_out, e->h_out, 0));
    memset(e->h_out, 0, e->out_bytes);
    CK(cudaMemset(e->d_out, 0, e->out_bytes));
    // small batches: the kernel reads actions from / writes results to mapped pinned host memory (no copy engine
    // round trips); large batches use bulk DMA copies.  MARO_B200_ZEROCOPY=0/1 overrides.
    const char* z = getenv("MARO_B200_ZEROCOPY");
    e->zero_copy = z ? atoi(z) != 0 : e->B <= 16384;
    return 0;
}

// Host-buffer step shared by the scenarios: stage inputs, run `step_device`, fetch outputs, synchronise.
// `pinned` = the caller filled / reads the library's pinned staging buffers directly (maro_*_pinned_buffers): the
// pointers are then only presence flags and no host-side memcpy happens.
template <class StepDevice>
static int common_host_step(EnvCommon* e, const uint8_t* active, const int32_t* actions, const int32_t* n_actions,
                            int32_t* decisions, int64_t* metrics, StepDevice step_device, bool pinned = false) {
    const int B = e->B, A = e->max_actions;
    const size_t act_bytes = (size_t)B * A * 16, nact_off = act_bytes, active_off = act_bytes + (size_t)B * 4;
    const size_t dec_bytes = (size_t)B * e->dec_words * 4;
    if (!pinned) {
        if (actions) memcpy(e->h_in, actions, act_bytes);
        if (actions && n_actions) memcpy(e->h_in + nact_off, n_actions, (size_t)B * 4);
        if (active) memcpy(e->h_in + active_off, active, B);
    }
    uint8_t* in = e->zero_copy ? e->hd_in : e->d_in;
    uint8_t* out = e->zero_copy ? e->hd_out : e->d_out;
    if (!e->zero_copy) {
        size_t lo = e->in_bytes, hi = 0;  // byte range of the staging buffer that must travel
        if (actions) { lo = 0; hi = act_bytes; }
        if (actions && n_actions) hi = nact_off + (size_t)B * 4;
        if (active) { lo = std::min(lo, active_off); hi = active_off + B; }
        if (hi > lo) CK(cudaMemcpyAsync(e->d_in + lo, e->h_in + lo, hi - lo, cudaMemcpyHostToDevice, e->stream));
    }
    int rc = step_device(active ? in + active_off : nullptr, actions ? reinterpret_cast<const int32_t*>(in) : nullptr,
                         actions && n_actions ? reinterpret_cast<const int32_t*>(in + nact_off) : nullptr,
                         reinterpret_cast<int32_t*>(out), reinterpret_cast<int64_t*>(out + dec_bytes));
    if (rc) return rc;
    if (!e->zero_copy) CK(cudaMemcpyAsync(e->h_out, e->d_out, e->out_bytes, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (!pinned) {
        memcpy(decisions, e->h_out, dec_bytes);
        memcpy(metrics, e->h_out + dec_bytes, (size_t)B * e->met_words * 8);
    }
    return 0;
}

// Reset masks go straight from the caller's bytes into the device-side active region of d_in.  The pinned staging buffers
// belong to the caller between steps (actions / n_actions / active filled for the next step_pinned, or read by a submit on
// another replica range), so a reset must not write them.  d_in's active region is private to the library: the bulk-copy
// step refills it before every use and the zero-copy step reads hd_in.  The caller synchronises the stream before
// returning, so a pageable mask is fine.
static int common_stage_mask(EnvCommon* e, const uint8_t* mask, const uint8_t** d_active) {
    uint8_t* dst = e->d_in + (size_t)e->B * e->max_actions * 16 + (size_t)e->B * 4;
    CK(cudaMemcpyAsync(dst, mask, e->B, cudaMemcpyHostToDevice, e->stream));
    *d_active = dst;
    return 0;
}

static int common_pinned_buffers(EnvCommon* e,void** actions, void** n_actions, void** active, void** decisions, void** metrics) {
    if (!e) return fail("pinned_buffers: null handle");
    const size_t B = (size_t)e->B, act_bytes = B * e->max_actions * 16;
    if (actions) *actions = e->h_in;
    if (n_actions) *n_actions = e->h_in + act_bytes;
    if (active) *active = e->h_in + act_bytes + B * 4;
    if (decisions) *decisions = e->h_out;
    if (metrics) *metrics = e->h_out + B * e->dec_words * 4;
    return 0;
}

static int common_read_frame(EnvCommon* e, int32_t replica, int32_t* out_words, int32_t n_words) {
    if (!e || replica < 0 || replica >= e->B || !out_words || n_words < e->FW) return fail("read_frame: bad arguments");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(out_words, e->d_state + (size_t)replica * e->SW, (size_t)e->FW * 4, cudaMemcpyDeviceToHost));
    return 0;
}
static int common_ticks(EnvCommon* e, int32_t* out_ticks) {
    if (!e || !out_ticks) return fail("ticks: bad arguments");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy2D(out_ticks, 4, e->d_state + e->off_tick, (size_t)e->SW * 4, 4, e->B, cudaMemcpyDeviceToHost));
    return 0;
}
static int common_counters(EnvCommon* e, int64_t* out) {
    if (!e || !out) return fail("counters: bad arguments");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy2D(out, 32, e->d_state + e->off_counters, (size_t)e->SW * 4, 32, e->B, cudaMemcpyDeviceToHost));
    return 0;
}
static int common_snapshot_frames(EnvCommon* e, int32_t replica, int32_t* out, int32_t cap, int32_t* n_out) {
    if (!e || replica < 0 || replica >= e->B || !out || !n_out) return fail("snapshot_frames: bad arguments");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    std::vector<int32_t> rows(e->ring_rows);
    CK(cudaMemcpy(rows.data(), e->d_snap_frame + (size_t)replica * e->ring_rows, rows.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<int32_t> have;
    for (int32_t f : rows) if (f >= 0) have.push_back(f);
    std::sort(have.begin(), have.end());
    *n_out = (int32_t)have.size();
    for (int i = 0; i < (int)have.size() && i < cap; i++) out[i] = have[i];
    return 0;
}
// ---- device-state checkpoint (SURVEY.md §8f rank 3: "enables env.dump / checkpoint of device state") -------------------
// File: CkptHeader | state [B][SW] i32 | snap_frame [B][ring] i32 | (snap [B][ring][FWp] i32 when with_snapshots) | extras.
// A checkpoint restores into a handle created with the same topology / configuration (the header's shape must match).
struct CkptHeader {
    char magic[8];
    int32_t version, scenario, B, SW, FWp, ring_rows, with_snapshots, n_extra;
    int64_t extra_bytes[8];
};

static int ckpt_copy(FILE* fp, void* d_ptr, size_t bytes, bool save, cudaStream_t stream) {
    const size_t chunk = 32u << 20;
    std::vector<uint8_t> host(std::min(bytes, chunk));
    for (size_t off = 0; off < bytes; off += chunk) {
        const size_t n = std::min(chunk, bytes - off);
        if (save) {
            CK(cudaMemcpyAsync(host.data(), (uint8_t*)d_ptr + off, n, cudaMemcpyDeviceToHost, stream));
            CK(cudaStreamSynchronize(stream));
            if (fwrite(host.data(), 1, n, fp) != n) return fail("checkpoint: short write");
        } else {
            if (fread(host.data(), 1, n, fp) != n) return fail("checkpoint: short read (truncated file)");
            CK(cudaMemcpyAsync((uint8_t*)d_ptr + off, host.data(), n, cudaMemcpyHostToDevice, stream));
            CK(cudaStreamSynchronize(stream));
        }
    }
    return 0;
}

static int common_save(EnvCommon* e, const char* path, int32_t with_snapshots) {
    if (!e || !path) return fail("save: bad arguments");
    if (e->ckpt_extra.size() > 8) return fail("save: too many extra buffers");
    CK(cudaSetDevice(e->device));
    FILE* fp = fopen(path, "wb");
    if (!fp) return fail(std::string("save: cannot open ") + path);
    CkptHeader h;
    memset(&h, 0, sizeof(h));
    memcpy(h.magic, "MAROB2CK", 8);
    h.version = 1; h.scenario = e->scenario_id; h.B = e->B; h.SW = e->SW; h.FWp = e->FWp; h.ring_rows = e->ring_rows;
    h.with_snapshots = with_snapshots ? 1 : 0; h.n_extra = (int32_t)e->ckpt_extra.size();
    for (size_t i = 0; i < e->ckpt_extra.size(); i++) h.extra_bytes[i] = *e->ckpt_extra[i].d_ptr ? (int64_t)e->ckpt_extra[i].bytes : 0;
    int rc = fwrite(&h, sizeof(h), 1, fp) == 1 ? 0 : fail("save: short write");
    const size_t B = (size_t)e->B;
    if (!rc) rc = ckpt_copy(fp, e->d_state, B * e->SW * 4, true, e->stream);
    if (!rc) rc = ckpt_copy(fp, e->d_snap_frame, B * e->ring_rows * 4, true, e->stream);
    if (!rc && with_snapshots) rc = ckpt_copy(fp, e->d_snap, B * e->ring_rows * e->FWp * 4, true, e->stream);
    for (size_t i = 0; !rc && i < e->ckpt_extra.size(); i++)
        if (h.extra_bytes[i]) rc = ckpt_copy(fp, *e->ckpt_extra[i].d_ptr, (size_t)h.extra_bytes[i], true, e->stream);
    if (fclose(fp) != 0 && !rc) rc = fail("save: close failed");
    return rc;
}

static int common_load(EnvCommon* e, const char* path) {
    if (!e || !path) return fail("load: bad arguments");
    CK(cudaSetDevice(e->device));
    FILE* fp = fopen(path, "rb");
    if (!fp) return fail(std::string("load: cannot open ") + path);
    CkptHeader h;
    int rc = 0;
    if (fread(&h, sizeof(h), 1, fp) != 1 || memcmp(h.magic, "MAROB2CK", 8) != 0 || h.version != 1) rc = fail("load: not a maro_b200 checkpoint");
    if (!rc && (h.scenario != e->scenario_id || h.B != e->B || h.SW != e->SW || h.FWp != e->FWp || h.ring_rows != e->ring_rows ||
                h.n_extra != (int32_t)e->ckpt_extra.size()))
        rc = fail("load: the checkpoint was written by a handle of a different shape (scenario / replicas / topology / snapshot ring)");
    for (size_t i = 0; !rc && i < e->ckpt_extra.size(); i++) {
        const int64_t have = *e->ckpt_extra[i].d_ptr ? (int64_t)e->ckpt_extra[i].bytes : 0;
        if (h.extra_bytes[i] != have) rc = fail(std::string("load: buffer '") + e->ckpt_extra[i].name + "' differs in size");
    }
    const size_t B = (size_t)e->B;
    if (!rc) rc = ckpt_copy(fp, e->d_state, B * e->SW * 4, false, e->stream);
    if (!rc) rc = ckpt_copy(fp, e->d_snap_frame, B * e->ring_rows * 4, false, e->stream);
    if (!rc) {
        if (h.with_snapshots) rc = ckpt_copy(fp, e->d_snap, B * e->ring_rows * e->FWp * 4, false, e->stream);
        else {  // rows were not saved: the ring restarts empty (queries of earlier frames read as "not held")
            CK(cudaMemsetAsync(e->d_snap_frame, 0xff, B * e->ring_rows * 4, e->stream));
            CK(cudaStreamSynchronize(e->stream));
        }
    }
    for (size_t i = 0; !rc && i < e->ckpt_extra.size(); i++)
        if (h.extra_bytes[i]) rc = ckpt_copy(fp, *e->ckpt_extra[i].d_ptr, (size_t)h.extra_bytes[i], false, e->stream);
    fclose(fp);
    return rc;
}

static int common_set_query_layout(EnvCommon* e, int32_t layout) {
    if (!e || (layout != 0 && layout != 1)) return fail("set_query_layout: layout must be 0 (static) or 1 (dynamic)");
    e->query_layout = layout;
    return 0;
}
static int32_t common_attr_id(EnvCommon* e, int32_t node_type, const char* name) {
    if (!e || node_type < 0 || node_type >= e->n_node_types || !name) return -1;
    for (size_t i = 0; i < e->attrs[node_type].size(); i++)
        if (!strcmp(e->attrs[node_type][i].name, name)) return (int32_t)i;
    return -1;
}
static int32_t common_attr_slots(EnvCommon* e, int32_t node_type, int32_t attr_id) {
    if (!e || node_type < 0 || node_type >= e->n_node_types || attr_id < 0 || attr_id >= (int)e->attrs[node_type].size()) return -1;
    return e->attrs[node_type][attr_id].slots;
}


static int query_impl(EnvCommon* e, const int32_t* replicas, int32_t nr, int32_t node_type, const int32_t* frames,
                      int32_t nf, const int32_t* nodes, int32_t nn, const int32_t* attrs, int32_t na, double* d_out,
                      double* h_out, int64_t* out_per_replica) {
    if (!e || node_type < 0 || node_type >= e->n_node_types || nr < 1 || nf < 1 || nn < 1 || na < 1 || !replicas || !frames || !nodes || !attrs)
        return fail("maro_cim_query: bad arguments");
    CK(cudaSetDevice(e->device));
    const auto& reg = e->attrs[node_type];
    std::vector<int32_t> idx;
    idx.reserve(nr + nf + nn + 4 * na);
    for (int i = 0; i < nr; i++) { if (replicas[i] < 0 || replicas[i] >= e->B) return fail("maro_cim_query: replica out of range"); idx.push_back(replicas[i]); }
    for (int i = 0; i < nf; i++) idx.push_back(frames[i]);
    for (int i = 0; i < nn; i++) { if (nodes[i] < 0 || nodes[i] >= reg[0].n_nodes) return fail("maro_cim_query: node index out of range"); idx.push_back(nodes[i]); }
    int prefix = 0, max_slots = 1;
    std::vector<int32_t> off(na), slots(na), isf(na), pre(na);
    for (int i = 0; i < na; i++) {
        if (attrs[i] < 0 || attrs[i] >= (int)reg.size()) return fail("maro_cim_query: attribute id out of range");
        off[i] = reg[attrs[i]].off; slots[i] = reg[attrs[i]].slots; isf[i] = reg[attrs[i]].isf; pre[i] = prefix;
        prefix += slots[i];
        max_slots = std::max(max_slots, slots[i]);
    }
    if (e->query_layout == 1) prefix = na * max_slots;
    idx.insert(idx.end(), off.begin(), off.end());
    idx.insert(idx.end(), slots.begin(), slots.end());
    idx.insert(idx.end(), isf.begin(), isf.end());
    idx.insert(idx.end(), pre.begin(), pre.end());
    if (idx.size() > e->qidx_cap) {
        cudaFree(e->d_qidx);
        e->qidx_cap = idx.size() * 2;
        CK(cudaMalloc(&e->d_qidx, e->qidx_cap * 4));
    }
    CK(cudaMemcpyAsync(e->d_qidx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, e->stream));
    const int64_t per_rep = (int64_t)nf * nn * prefix, total = per_rep * nr;
    if (out_per_replica) *out_per_replica = per_rep;
    double* dst = d_out;
    if (!dst) {
        if ((size_t)total > e->qout_cap) {
            cudaFree(e->d_qout);
            e->qout_cap = (size_t)total * 2;
            CK(cudaMalloc(&e->d_qout, e->qout_cap * 8));
        }
        dst = e->d_qout;
    }
    QueryArgs q;
    q.snap = e->d_snap; q.snap_frame = e->d_snap_frame;
    q.replicas = e->d_qidx; q.frames = q.replicas + nr; q.nodes = q.frames + nf;
    q.attr_off = q.nodes + nn; q.attr_slots = q.attr_off + na; q.attr_isf = q.attr_slots + na; q.attr_prefix = q.attr_isf + na;
    q.nr = nr; q.nf = nf; q.nn = nn; q.na = na; q.slots_per_node = prefix; q.ring_rows = e->ring_rows; q.FWp = e->FWp;
    q.layout = e->query_layout; q.max_slots = max_slots;
    q.out = dst;
    int threads = 256;
    int blocks = (int)std::min<int64_t>((total + threads - 1) / threads, (int64_t)e->n_sm * 8);
    cim_query_kernel<<<blocks, threads, 0, e->stream>>>(q);
    CK(cudaGetLastError());
    if (h_out) CK(cudaMemcpyAsync(h_out, dst, (size_t)total * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));  // idx vector must outlive the async H2D
    return 0;
}

