// TEST INFRASTRUCTURE ONLY — the host emulator (emul.cpp) plus the small-topology instantiation of the CIM step,
// replica_step<G, false, kSmall = true>, run the way the resident kernel runs it: control state loaded into Ctl, one step,
// stored back.  Built by tests/test_kernel_logic_emulated_small.py into tests/_emul; never loaded by the package.
#include "emul.cpp"

template <int G>
static void small_step_g(Emul* e, int i, const int32_t* actp, int n, int32_t* dec, int64_t* met) {
    Replica r = rep_of(e, i);
    if (n > G) n = G;
    wemu::run_group(G, [&](int lane) {
        Act4 act = {0, 0, 0, 0};
        if (lane < n) { act.v = actp[4 * lane]; act.p = actp[4 * lane + 1]; act.qty = actp[4 * lane + 2]; act.type = actp[4 * lane + 3]; }
        Ctl k;
        ctl_load<G, true>(e->s, Grp<G>(lane), r, k);
        replica_step<G, false, true>(e->s, Grp<G>(lane), r, k, act, n, dec, met);
        ctl_store<G, true>(e->s, Grp<G>(lane), r, k);
    });
}

extern "C" {
// one env-step of every replica through the small-topology instantiation; returns 0 (and steps nothing) where
// cim_small_ok refuses the shape at the handle's lane width
int emul_small_step(Emul* e, const int32_t* actions, const int32_t* n_actions, int32_t* decisions, int64_t* metrics) {
    if (!cim_small_ok(e->s, e->lanes)) return 0;
    for (int i = 0; i < e->B; i++) {
        int n = actions ? (n_actions ? n_actions[i] : 1) : 0;
        const int32_t* act = actions ? actions + (size_t)i * e->s.max_actions * 4 : nullptr;
        int32_t* dec = decisions + (size_t)i * e->s.DW;
        int64_t* met = metrics + i * 3;
        switch (e->lanes) {
            case 8: small_step_g<8>(e, i, act, n, dec, met); break;
            case 16: small_step_g<16>(e, i, act, n, dec, met); break;
            default: small_step_g<32>(e, i, act, n, dec, met); break;
        }
    }
    return 1;
}
int emul_small_ok(Emul* e) { return cim_small_ok(e->s, e->lanes) ? 1 : 0; }
int emul_due_ring_slots(Emul* e) { return e->s.due_R; }  // 0: discharges go through the calendar queue
}
