// cim_host.hpp — host-side (plain C++) shape + static-table serialisation shared by cim_env.cu and the
// test-only host-emulation harness (tests/_emul).  No CUDA here.
#pragma once
#include <math.h>
#include <cmath>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/maro_b200.h"
#include "cim_core.cuh"

namespace maro {

inline void mt_init_by_array(uint32_t seed, uint32_t* mt) {
    mt[0] = 19650218u;
    for (int i = 1; i < 624; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    int i = 1, j = 0;
    for (int k = 624; k; k--) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + seed + (uint32_t)j;
        i++; j++;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
        if (j >= 1) j = 0;
    }
    for (int k = 623; k; k--) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
        i++;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
    }
    mt[0] = 0x80000000u;
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct BlobBuilder {
    std::vector<int32_t>& w;
    explicit BlobBuilder(std::vector<int32_t>& v) : w(v) {}
    int put_i(const int32_t* p, int n, int reserve) {
        int off = (int)w.size();
        w.insert(w.end(), p, p + n);
        w.resize(off + std::max(reserve, n), 0);
        return off;
    }
    int put_d(const double* p, int n, int reserve) {
        if (w.size() & 1) w.push_back(0);
        int off = (int)w.size();
        w.resize(off + 2 * std::max(reserve, n), 0);
        memcpy(w.data() + off, p, sizeof(double) * n);
        return off;
    }
};

// builtin sum() of floats as CPython >= 3.12 evaluates it (Neumaier compensated; see py_sum in cim_core.cuh)
inline double py_sum_host(const std::vector<double>& x) {
    if (x.empty()) return 0.0;
    double f = 0.0 + x[0], c = 0.0;
    for (size_t i = 1; i < x.size(); i++) {
        double v = x[i], t = f + v;
        if (fabs(f) >= fabs(v)) c += (f - t) + v; else c += (v - t) + f;
        f = t;
    }
    if (c != 0.0 && std::isfinite(c)) f += c;
    return f;
}

// Order list of one tick for a noise-free, fixed-mode topology: the arithmetic of
// CimSyntheticDataContainer._gen_orders (cim_data_container.py:310-398) with every noise term == 0.
inline void gen_orders_noise_free(const MaroCimTopology& t, int orders_to_gen, std::vector<int32_t>& out) {
    const int P = t.n_ports;
    int remaining = orders_to_gen;
    std::vector<double> tmp;
    for (int p = 0; p < P; p++) tmp.push_back(t.source_base[p] + 0.0);
    const double tot = py_sum_host(tmp);
    for (int p = 0; p < P; p++) {
        if (remaining == 0) break;
        int lo = t.target_offset[p], hi = t.target_offset[p + 1];
        tmp.clear();
        for (int i = lo; i < hi; i++) tmp.push_back(t.target_base[i] + 0.0);
        const double ttot = py_sum_host(tmp);
        double sp = t.source_base[p] + 0.0;
        if (tot != 0.0) sp = sp / tot;
        int cur = (int)ceil((double)orders_to_gen * sp);
        if (cur > remaining) cur = remaining;
        remaining -= cur;
        if (cur > 0) {
            int trem = cur;
            for (int i = lo; i < hi; i++) {
                double tp = t.target_base[i] + 0.0;
                if (ttot != 0.0) tp = tp / ttot;
                int num = (int)ceil((double)cur * tp);
                if (num > trem) num = trem;
                trem -= num;
                if (num > 0) {
                    out.push_back(p | (t.target_port[i] << 8));
                    out.push_back(num);
                }
            }
        }
    }
}

inline int count_distinct_orders(const MaroCimTopology& t) {
    std::vector<int32_t> v(t.order_proportion, t.order_proportion + t.max_tick);
    std::sort(v.begin(), v.end());
    return (int)(std::unique(v.begin(), v.end()) - v.begin());
}

// Serialise one topology into a blob; every array is padded to the per-handle maxima so that all topologies of
// a handle share the same offsets (CimShape::t_*).
inline int build_blob(const MaroCimTopology& t, CimShape& s, std::vector<int32_t>& out, int max_stops, int max_targets,
                      bool first, int max_distinct = 0) {
    std::vector<int32_t> w;
    BlobBuilder b(w);
    const int P = t.n_ports, V = t.n_vessels;
    CimShape o = s;
    o.t_port_capacity = b.put_i(t.port_capacity, P, P);
    o.t_port_init_empty = b.put_i(t.port_init_empty, P, P);
    o.t_frb_d = b.put_d(t.full_return_base, P, P);
    o.t_frn_d = b.put_d(t.full_return_noise, P, P);
    o.t_erb_d = b.put_d(t.empty_return_base, P, P);
    o.t_ern_d = b.put_d(t.empty_return_noise, P, P);
    o.t_sb_d = b.put_d(t.source_base, P, P);
    o.t_sn_d = b.put_d(t.source_noise, P, P);
    o.t_target_offset = b.put_i(t.target_offset, P + 1, P + 1);
    const int nt = t.target_offset[P];
    o.t_target_port = b.put_i(t.target_port, nt, max_targets);
    o.t_tb_d = b.put_d(t.target_base, nt, max_targets);
    o.t_tn_d = b.put_d(t.target_noise, nt, max_targets);
    o.t_vessel_capacity = b.put_i(t.vessel_capacity, V, V);
    o.t_vessel_init_empty = b.put_i(t.vessel_init_empty, V, V);
    o.t_vessel_route = b.put_i(t.vessel_route, V, V);
    o.t_vessel_period = b.put_i(t.vessel_period, V, V);
    o.t_vessel_route_start = b.put_i(t.vessel_route_start, V, V);
    o.t_vessel_leg_offset = b.put_i(t.vessel_leg_offset, V + 1, V + 1);
    o.t_vessel_leg = b.put_i(t.vessel_leg, t.vessel_leg_offset[V], t.vessel_leg_offset[V]);
    o.t_stop_offset = b.put_i(t.stop_offset, V + 1, V + 1);
    const int ns = t.stop_offset[V];
    o.t_stop_arrival = b.put_i(t.stop_arrival, ns, max_stops);
    o.t_stop_leave = b.put_i(t.stop_leave, ns, max_stops);
    o.t_stop_port = b.put_i(t.stop_port, ns, max_stops);
    o.t_route_offset = b.put_i(t.route_offset, t.n_routes + 1, t.n_routes + 1);
    o.t_route_port = b.put_i(t.route_port, t.route_offset[t.n_routes], t.route_offset[t.n_routes]);
    o.t_order_proportion = b.put_i(t.order_proportion, t.max_tick, t.max_tick);
    uint32_t mt[624];
    mt_init_by_array(t.order_number_seed, mt);
    o.t_mt_order = b.put_i(reinterpret_cast<int32_t*>(mt), 624, 624);
    mt_init_by_array(t.buffer_time_seed, mt);
    o.t_mt_buffer = b.put_i(reinterpret_cast<int32_t*>(mt), 624, 624);
    {   // integer buffer ticks (valid when the buffer stream is noise-free)
        std::vector<int32_t> fi(P), ei(P);
        for (int p = 0; p < P; p++) {
            fi[p] = (int)ceil(t.full_return_base[p] + 0.0);
            ei[p] = (int)ceil(t.empty_return_base[p] + 0.0);
        }
        o.t_frb_i = b.put_i(fi.data(), P, P);
        o.t_erb_i = b.put_i(ei.data(), P, P);
    }
    if (s.order_table) {
        std::vector<int32_t> vals(t.order_proportion, t.order_proportion + t.max_tick);
        std::sort(vals.begin(), vals.end());
        vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
        std::vector<int32_t> slot(t.max_tick), off(1, 0), list;
        for (int k = 0; k < t.max_tick; k++)
            slot[k] = (int)(std::lower_bound(vals.begin(), vals.end(), t.order_proportion[k]) - vals.begin());
        for (int32_t v : vals) {
            gen_orders_noise_free(t, v, list);
            off.push_back((int)list.size() / 2);
        }
        o.t_ord_slot = b.put_i(slot.data(), t.max_tick, t.max_tick);
        o.t_ord_off = b.put_i(off.data(), (int)off.size(), max_distinct + 1);
        o.t_ord_list = b.put_i(list.data(), (int)list.size(), 2 * max_distinct * std::max(1, max_targets));
    }
    w.resize(round_up((int)w.size(), 4), 0);
    o.table_words = (int)w.size();
    if (first) s = o;
    else if (o.table_words != s.table_words || o.t_mt_buffer != s.t_mt_buffer) return 1;
    out.insert(out.end(), w.begin(), w.end());
    return 0;
}

inline int check_same_shape(const MaroCimTopology& a, const MaroCimTopology& b) {
    if (a.n_ports != b.n_ports || a.n_vessels != b.n_vessels || a.n_routes != b.n_routes ||
        a.past_stop_number != b.past_stop_number || a.future_stop_number != b.future_stop_number ||
        a.max_tick != b.max_tick || a.order_mode != b.order_mode || a.container_volume != b.container_volume ||
        a.total_containers != b.total_containers)
        return 1;
    for (int i = 0; i <= a.n_routes; i++)
        if (a.route_offset[i] != b.route_offset[i]) return 1;
    for (int i = 0; i <= a.n_ports; i++)
        if (a.target_offset[i] != b.target_offset[i]) return 1;
    return 0;
}


// Fill `s` (layout, queue sizing) and serialise every topology into `tables`.  Returns non-zero on mismatch.
// What one topology instance asks of a handle's sizing: the longest event delay (calendar-queue horizon), the buffer
// ticks behind the default queue capacity, and which MT19937 streams it draws from.
// `stops_increase`: every vessel visits its stops at strictly increasing ticks (the condition of the due rings).
struct CimTopoNeeds {
    int max_delay = 2, buf_full = 1, buf_empty = 1, max_stops = 0;
    bool order_noise = false, buffer_noise = false, stops_increase = true;
};
inline CimTopoNeeds topology_needs(const MaroCimTopology& t) {
    CimTopoNeeds n;
    const int P = t.n_ports, V = t.n_vessels;
    n.max_stops = t.stop_offset[V];
    for (int v = 0; v < V; v++)
        for (int i = t.stop_offset[v] + 1; i < t.stop_offset[v + 1]; i++)
            if (t.stop_arrival[i] <= t.stop_arrival[i - 1]) n.stops_increase = false;
    for (int p = 0; p < P; p++) {
        if (t.source_noise[p] != 0) n.order_noise = true;
        if (t.full_return_noise[p] != 0 || t.empty_return_noise[p] != 0) n.buffer_noise = true;
        n.buf_full = std::max(n.buf_full, (int)ceil(t.full_return_base[p] + fabs(t.full_return_noise[p])));
        n.buf_empty = std::max(n.buf_empty, (int)ceil(t.empty_return_base[p] + fabs(t.empty_return_noise[p])));
    }
    for (int i = 0; i < t.target_offset[P]; i++)
        if (t.target_noise[i] != 0) n.order_noise = true;
    for (int v = 0; v < V; v++) {
        int rl = t.route_offset[t.vessel_route[v] + 1] - t.route_offset[t.vessel_route[v]];
        for (int i = t.stop_offset[v]; i < t.stop_offset[v + 1]; i++) {
            int j = std::min(i + rl, t.stop_offset[v + 1] - 1);
            n.max_delay = std::max(n.max_delay, t.stop_arrival[j] - t.stop_arrival[i] + 1);
        }
    }
    n.max_delay = std::max(n.max_delay, std::max(n.buf_full, n.buf_empty) + 1);
    return n;
}

inline int compute_shape_and_tables(const MaroCimTopology* topos, int n_topos, const MaroCimConfig* cfg, CimShape& s,
                                    std::vector<int32_t>& tables, int& max_stops_out, int& max_targets_out,
                                    int& max_distinct_out) {
    const MaroCimTopology& t0 = topos[0];
    memset(&s, 0, sizeof(s));
    const int P = t0.n_ports, V = t0.n_vessels;
    s.P = P; s.V = V; s.R = t0.n_routes; s.past = t0.past_stop_number; s.fut = t0.future_stop_number;
    s.max_tick = t0.max_tick; s.start_tick = cfg->start_tick;
    s.resolution = cfg->snapshot_resolution > 0 ? cfg->snapshot_resolution : 1;
    const int durations = s.max_tick - s.start_tick;
    if (durations < 1) return 1;
    const int total_frames = (durations + s.resolution - 1) / s.resolution;
    s.ring_rows = cfg->max_snapshots > 0 ? std::min(cfg->max_snapshots, total_frames) : total_frames;
    s.order_mode = t0.order_mode; s.total_containers = t0.total_containers; s.vol = t0.container_volume;
    s.max_actions = cfg->max_actions > 0 ? cfg->max_actions : 1;
    s.n_replicas = cfg->n_replicas;
    s.joint = cfg->decision_mode == 1 ? 1 : 0;
    s.DW = s.joint ? MARO_CIM_DECISION_WORDS * V : MARO_CIM_DECISION_WORDS;
    if (s.joint && s.max_actions < V) s.max_actions = V;  // one answer row per decision event of a tick
    int max_stops = 0, max_targets = t0.target_offset[P], max_delay = 2, max_rl = 1, buf_full = 1, buf_empty = 1;
    bool stops_increase = true;
    for (int r = 0; r < t0.n_routes; r++) max_rl = std::max(max_rl, t0.route_offset[r + 1] - t0.route_offset[r]);
    s.max_route_len = max_rl;
    for (int k = 0; k < n_topos; k++) {
        const CimTopoNeeds n = topology_needs(topos[k]);
        stops_increase = stops_increase && n.stops_increase;
        max_stops = std::max(max_stops, n.max_stops);
        if (n.order_noise) s.order_noise = 1;
        if (n.buffer_noise) s.buffer_noise = 1;
        buf_full = std::max(buf_full, n.buf_full);
        buf_empty = std::max(buf_empty, n.buf_empty);
        max_delay = std::max(max_delay, n.max_delay);
    }
    // re-seeded instances of the same config (Env.reset(keep_seed=False), set_seed) draw other vessel speeds / parking
    // times: 25 % head-room on the horizon; maro_cim_set_topology re-validates every replacement against it
    max_delay += max_delay / 4 + 8;
    // frame layout (DESIGN.md "Frame layout")
    s.o_vs = 12 * P;
    s.o_past = s.o_vs + 10 * V;
    s.o_past_tick = s.o_past + V * s.past;
    s.o_fut = s.o_past_tick + V * s.past;
    s.o_fut_tick = s.o_fut + V * s.fut;
    s.o_fop = s.o_fut_tick + V * s.fut;
    s.o_fov = s.o_fop + P * P;
    s.o_vp = s.o_fov + V * P;
    s.FW = s.o_vp + V * P;
    s.FWp = round_up(s.FW, 4);
    // delay lines for the pure-add events of noise-free, small topologies (cim_core.cuh: CimShape::DL): sized for the longest
    // container buffer time; the calendar queue then only carries DISCHARGE_FULL.  MARO_B200_DELAY_LINE=0 turns them off (A/B).
    int dl = 2;
    while (dl < std::max(buf_full, buf_empty) + 1) dl <<= 1;
    const int dl_stride = round_up(P * P + P + 2, 4);
    const char* dl_off = getenv("MARO_B200_DELAY_LINE");
    const bool noise_free = !s.order_noise && s.order_mode == 0 && !s.buffer_noise;
    const bool dl_on = noise_free && dl * dl_stride <= 512 && !(dl_off && atoi(dl_off) == 0);
    // due rings for DISCHARGE_FULL where every vessel's stop ticks increase strictly (CimShape::due_R): the calendar queue is
    // then not used at all and keeps no slots or buckets
    if (dl_on && stops_increase) {
        s.due_R = 1;
        while (s.due_R < max_rl + 1) s.due_R <<= 1;
    }
    s.CWp = round_up(C_FIXED + (s.due_R ? 5 : 3) * V, 4);
    if (s.due_R) {
        s.QH = 0;
        s.QN = 0;
    } else {
        int qh = 16;
        while (qh < max_delay + 1) qh <<= 1;
        s.QH = qh;
        // outstanding dynamic events: RETURN_FULL <= orders/tick x buffer, DISCHARGE_FULL <= V x route, RETURN_EMPTY
        int qn = cfg->queue_capacity > 0 ? cfg->queue_capacity
                                         : std::max(32, max_targets * buf_full + V * max_rl * (1 + buf_empty));
        if (qn > 65000) qn = 65000;
        s.QN = round_up(qn, 4);
    }
    s.SW = round_up(s.FWp + s.CWp + s.QN * 2 + s.QH + s.QN, 4);  // frame | ctrl | ev | buckets | next+free (u16)
    if (dl_on) {
        s.DL = dl; s.dl_stride = dl_stride; s.o_dl = s.SW;  // (word offset from the start of the block = from r.f)
        s.SW = round_up(s.SW + dl * dl_stride, 4);
    }
    if (s.due_R) {
        s.o_due = s.SW;
        s.SW = round_up(s.SW + 2 * V * s.due_R, 4);
    }
    s.res_is_one = s.resolution == 1 ? 1 : 0;
    s.vol_is_one = s.vol == 1.0 ? 1 : 0;
    s.max_targets = max_targets;
    s.mt_scratch = 2 * 640;
    // tables (stop arrays get 12.5% head-room so that re-seeded topologies of the same config still fit)
    max_stops += max_stops / 8 + 8;
    max_stops_out = max_stops;
    max_targets_out = max_targets;
    s.order_table = (!s.order_noise && s.order_mode == 0) ? 1 : 0;
    int max_distinct = 0;
    if (s.order_table)
        for (int k = 0; k < n_topos; k++) max_distinct = std::max(max_distinct, count_distinct_orders(topos[k]));
    max_distinct_out = max_distinct;
    tables.clear();
    for (int k = 0; k < n_topos; k++) {
        if (k > 0 && check_same_shape(t0, topos[k])) return 1;
        if (build_blob(topos[k], s, tables, max_stops, max_targets, k == 0, max_distinct)) return 1;
    }
    return 0;
}

// words of one replica's MT block: 2 states | 64 tail scratch | order list | float64 scratch
inline int mt_block_words(const CimShape& s) {
    int mt_even = (s.max_targets + 1) & ~1;
    // 2 MT states | 64 tail scratch | order list (2 words / target) | doubles srcd[P] tgtd[T] | ints cur[P] c2[T] cnt[P]
    return round_up(2 * 640 + 64 + 2 * mt_even + 2 * (s.P + mt_even) + (2 * s.P + mt_even) + 2 + 16, 4);
}

// lanes per replica: smallest power of two >= the widest cooperative phase of the topology (>= 8)
inline int lanes_per_replica(const CimShape& s) {
    int w = std::max(std::max(s.P, s.V), std::max(s.max_route_len, std::max(s.fut, s.past)));
    return w <= 8 ? 8 : (w <= 16 ? 16 : 32);
}

// May replica_step<G, false, kSmall = true> run this shape with G lanes per replica?  Noise-free fixed-order mode with
// integer buffer ticks (the kGeneral = false path), snapshot resolution 1, container volume 1, Sequential mode, delay
// lines and due rings on, and every dimension a lane loop runs over (ports, vessels, route stops, future stops) <= G.
inline bool cim_small_ok(const CimShape& s, int G) {
    return s.order_table && !s.order_noise && !s.buffer_noise && s.res_is_one && s.vol_is_one && !s.joint && s.DL > 0 && s.due_R > 0 &&
           s.P <= G && s.V <= G && s.max_route_len <= G && s.fut <= G;
}

}  // namespace maro
