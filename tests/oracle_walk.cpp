/*
 * Test infrastructure, NOT product code: RAPID_DELIVERY_SHUFFLED_BATCHES over the oracle's literal handlers, linear in the work.
 *
 * Compiled by tests/shuffled_ref.py together with oracle/oracle_capi.cpp (included unchanged, for the handle types), so that it
 * takes the orc_sim handles oracle/oracle_py.py creates.  Each receiver r of the sim walks the n batches of a sequence in its own
 * order P_g (g = receiver_base + r; the pseudocode next to RAPID_DELIVERY_SHUFFLED_BATCHES in include/rapid_b200.h, restated here
 * a third time) through its own AlertBatchHandler::handleBatch — MembershipService.handleMessage, gating included — and stops
 * after the batch it announces in.
 */
#include "../oracle/oracle_capi.cpp"

namespace {

struct Order {
    uint64_t key, m;
    int64_t n;
    int w;
    Order(uint64_t seed, int64_t g, int64_t n_) : key(splitmix64(seed + (uint64_t)g)), n(n_), w(4) {
        while (((int64_t)1 << (2 * w)) < n) ++w;
        m = ((uint64_t)1 << w) - 1;
    }
    uint64_t E(uint64_t v) const {
        uint64_t a = v >> w, b = v & m;
        for (int i = 0; i < 4; ++i) {
            const uint64_t t = a ^ (splitmix64(key ^ ((uint64_t)(i + 1) << 58) ^ b) & m);
            a = b;
            b = t;
        }
        return (a << w) | b;
    }
    int64_t at(int64_t j) const {
        if (n <= 1) return j;
        uint64_t v = E((uint64_t)j);
        while (v >= (uint64_t)n) v = E(v);
        return (int64_t)v;
    }
};

}  // namespace

extern "C" {

void wk_batch_order(uint64_t seed, int64_t g, int64_t n, int64_t* out) {
    const Order o(seed, g, n);
    for (int64_t j = 0; j < n; ++j) out[j] = o.at(j);
}

/* out_len[R] / out_ids: the proposal announced during this call (canonical order), out_in[R]: its batch index (-1: none),
 * out_announced[R]: announcedProposal after the call.  Returns the ids written, -1 if out_cap is too small. */
int64_t wk_apply_batches(orc_sim* s, int64_t A, const int32_t* src, const int32_t* dst, const uint8_t* ring, const uint8_t* status,
                         const int64_t* cfg, int64_t n_batches, const int64_t* off, const uint8_t* blocked, uint64_t seed,
                         int64_t receiver_base, int32_t n_threads, int32_t* out_len, uint8_t* out_announced, int32_t* out_in,
                         int32_t* out_ids, int64_t out_cap) {
    const orc_universe* u = s->view->u;
    MembershipView& view = *s->view->v;
    std::vector<std::vector<AlertMessage>> batches((size_t)n_batches);
    for (int64_t b = 0; b < n_batches; ++b)
        for (int64_t i = off[b]; i < off[b + 1]; ++i) {
            AlertMessage m;
            m.edgeSrc = u->eps[(size_t)src[i]];
            m.edgeDst = u->eps[(size_t)dst[i]];
            m.edgeStatus = status[i];
            m.configurationId = cfg[i];
            m.ringNumber.assign(1, (int32_t)ring[i]);
            batches[(size_t)b].push_back(m);
        }
    // the view's memo caches are filled single-threaded, as orc_sim_apply_batch does, so that the workers only read them
    view.getCurrentConfigurationId();
    for (int64_t i = 0; i < A; ++i) {
        const Endpoint& d = u->eps[(size_t)dst[i]];
        view.getRingZeroComparator().hashOf(d);
        if (view.isHostPresent(d)) view.getObserversOf(d);
        else { for (int k = 0; k < view.K(); ++k) view.comparator(k).hashOf(d); }
    }
    const int64_t R = s->R;
    std::vector<std::vector<Endpoint>> props((size_t)R);
    std::atomic<int64_t> next(0);
    auto worker = [&]() {
        for (;;) {
            const int64_t r = next.fetch_add(1);
            if (r >= R) break;
            out_in[r] = -1;
            if (blocked && blocked[r]) continue;
            AlertBatchHandler& h = *s->nodes[(size_t)r];
            const Order o(seed, receiver_base + r, n_batches);
            for (int64_t j = 0; j < n_batches && !h.announcedProposal(); ++j) {
                const int64_t b = o.at(j);
                std::vector<Endpoint> p = h.handleBatch(batches[(size_t)b]);
                if (!p.empty()) { props[(size_t)r] = std::move(p); out_in[r] = (int32_t)b; }
            }
        }
    };
    const int nt = n_threads < 1 ? 1 : n_threads;
    if (nt == 1) worker();
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < nt; ++t) th.emplace_back(worker);
        for (auto& t : th) t.join();
    }
    int64_t w = 0;
    for (int64_t r = 0; r < R; ++r) {
        out_len[r] = (int32_t)props[(size_t)r].size();
        out_announced[r] = s->nodes[(size_t)r]->announcedProposal() ? 1 : 0;
        for (const Endpoint& e : props[(size_t)r]) {
            if (w >= out_cap) return -1;
            out_ids[w++] = u->tagOf(e);
        }
    }
    return w;
}

}  // extern "C"
