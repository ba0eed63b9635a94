// whmec_heuristic_batch (DESIGN §4.10): many heuristic tables in one call.  Every table is prepared by the constructor part
// of heuristic.cpp; the tables the device can take are sized, cut into groups under the free HBM and swept one CTA per table
// (heuristic.cu); the output pass of heuristic.cpp turns each table's bipartition and transmission vector into the result.
// Every other table, and every table the device hands back, runs whmec_heuristic inside the call.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <numeric>
#include <string>
#include <vector>

#include "heuristic_batch.h"

namespace whmec {

namespace {

uint64_t align16(uint64_t x) { return (x + 15) & ~(uint64_t)15; }

// Byte offsets of the slices of one table, in one fixed order for heur_layout, heur_pack and heur_bind.
struct InSlices {
    uint64_t rc, mc, ev, read_off, ent_col, last, sample, start, gt, trios, seen, total;
};
struct WorkSlices {
    uint64_t votes[2], side[2], placed[2], tv[2], score[2], mut[2], from[2];
    uint64_t ht, a[4], best, f0, f1, add, equal_to, active, kept, back, rtv, rplaced, total;
};
struct OutSlices {
    uint64_t part, tv, status, total;
};

struct Carver {
    uint64_t at = 0;
    uint64_t take(uint64_t bytes) {
        const uint64_t o = at;
        at = align16(at + bytes);
        return o;
    }
};

InSlices in_slices(const HeurLayout &L) {
    Carver c;
    InSlices s;
    s.rc = c.take(4ull * L.n);
    s.mc = c.take(4ull * L.n);
    s.ev = c.take(4 * L.nnz);
    s.read_off = c.take(4ull * (L.m + 1));
    s.ent_col = c.take(4 * L.nnz);
    s.last = c.take(4ull * L.m);
    s.sample = c.take(4ull * L.m);
    s.start = c.take(4ull * (L.n + 1));
    s.gt = c.take((uint64_t)L.S * L.n);
    s.trios = c.take(12ull * L.n_trios);
    s.seen = c.take(L.S);
    s.total = c.at;
    return s;
}

WorkSlices work_slices(const HeurLayout &L) {
    Carver c;
    WorkSlices s;
    const uint64_t cap = L.cap;
    for (int b = 0; b < 2; ++b) {
        s.votes[b] = c.take(4 * cap * 2 * L.S * L.Wmax);
        s.side[b] = c.take(cap * L.Amax);
        s.placed[b] = c.take(cap * L.NNmax);
        s.tv[b] = c.take(4 * cap);
        s.score[b] = c.take(4 * cap);
        s.mut[b] = c.take(4 * cap);
        s.from[b] = c.take(4 * cap);
    }
    s.ht = c.take(4ull * L.ht_size);
    for (int i = 0; i < 4; ++i) s.a[i] = c.take(4 * cap);
    s.best = c.take(8 * cap);
    s.f0 = c.take(4 * cap);
    s.f1 = c.take(4 * cap);
    s.add = c.take(4ull * L.NNmax * L.Wmax);
    s.equal_to = c.take(4ull * L.NNmax);
    s.active = c.take(4ull * L.Amax);
    s.kept = c.take(4ull * L.Amax);
    s.back = c.take(2ull * L.n * L.rcap);
    s.rtv = c.take(4ull * L.n * L.rcap);
    s.rplaced = c.take((uint64_t)L.rcap * L.m);
    s.total = c.at;
    return s;
}

OutSlices out_slices(const HeurLayout &L) {
    Carver c;
    OutSlices s;
    s.part = c.take(L.m);
    s.tv = c.take(4ull * L.n);
    s.status = c.take(4);
    s.total = c.at;
    return s;
}

void set_err(char *errs, size_t errlen, uint32_t t, const std::string &msg) {
    if (errs && errlen) {
        char *e = errs + (size_t)t * errlen;
        std::strncpy(e, msg.c_str(), errlen - 1);
        e[errlen - 1] = 0;
    }
}

}  // namespace

bool heur_device_table(const HeurTable &tb) {
    return tb.allow_mut && tb.n > 0 && tb.m > 0 && tb.S > 0 && tb.S <= HEUR_MAX_S &&
           tb.p->read_off[tb.m] - tb.p->read_off[0] < 0xFFFFFFFFull;
}

HeurLayout heur_layout(const HeurTable &tb, uint32_t row_limit) {
    HeurLayout L;
    L.n = tb.n;
    L.m = tb.m;
    L.S = tb.S;
    L.n_trios = tb.n_trios;
    L.row_limit = row_limit;
    L.distrust = tb.distrust;
    L.nnz = tb.p->read_off[tb.m] - tb.p->read_off[0];
    const uint64_t rl = std::max<uint32_t>(row_limit, 1);
    L.cap = (uint32_t)std::min<uint64_t>(HEUR_MAX_CAP, std::max<uint64_t>(64, 2 * rl * (tb.n_trios ? 4 : 2)));
    L.rcap = (uint32_t)std::min<uint64_t>(L.cap, std::max<uint64_t>(64, 2 * rl));
    L.ht_size = 1;
    while (L.ht_size < 2 * L.cap) L.ht_size <<= 1;
    // window widths, active reads and new reads per column, as the sweep meets them
    uint32_t right = 0;
    std::vector<uint32_t> ends(tb.n + 1, 0);  // reads whose last column is k
    for (uint32_t r = 0; r < tb.m; ++r) ++ends[tb.last[r]];
    uint64_t active = 0;
    L.Wmax = 1;
    for (uint32_t col = 0; col < tb.n; ++col) {
        const uint32_t s0 = tb.start[col], s1 = tb.start[col + 1];
        right = std::max(right, col);
        for (uint32_t r = s0; r < s1; ++r) right = std::max(right, tb.last[r]);
        L.Wmax = std::max(L.Wmax, right + 1 - col);
        L.NNmax = std::max(L.NNmax, s1 - s0);
        active += s1 - s0;  // reads with first <= col <= last
        L.Amax = std::max<uint32_t>(L.Amax, (uint32_t)active);
        active -= ends[col];
    }
    L.Amax = std::max<uint32_t>(L.Amax, 1);
    L.NNmax = std::max<uint32_t>(L.NNmax, 1);
    L.in_bytes = in_slices(L).total;
    L.work_bytes = work_slices(L).total;
    L.out_bytes = out_slices(L).total;
    L.work = (uint64_t)tb.n * rl;
    return L;
}

std::vector<HeurGroup> heur_groups(std::vector<HeurLayout> &layouts, uint64_t budget, std::vector<uint32_t> &alone) {
    std::vector<uint32_t> order(layouts.size());
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return layouts[a].work > layouts[b].work; });
    std::vector<HeurGroup> groups;
    HeurGroup g;
    uint64_t used = 0;
    auto close = [&] {
        if (g.members.empty()) return;
        // offsets: the descriptors first, then every member's inputs; work and outputs in member order
        uint64_t in_at = align16(g.members.size() * sizeof(HeurDevTable)), work_at = 0, out_at = 0;
        for (uint32_t i : g.members) {
            HeurLayout &L = layouts[i];
            L.in_off = in_at;
            L.work_off = work_at;
            L.out_off = out_at;
            in_at += L.in_bytes;
            work_at += L.work_bytes;
            out_at += L.out_bytes;
        }
        g.in_bytes = in_at;
        g.work_bytes = work_at;
        g.out_bytes = out_at;
        groups.push_back(std::move(g));
        g = HeurGroup();
        used = 0;
    };
    for (uint32_t i : order) {
        const HeurLayout &L = layouts[i];
        const uint64_t bytes = L.in_bytes + L.work_bytes + L.out_bytes + sizeof(HeurDevTable) + 16;
        if (bytes > budget) {
            alone.push_back(i);
            continue;
        }
        if (used + bytes > budget) close();
        g.members.push_back(i);
        used += bytes;
    }
    close();
    return groups;
}

void heur_pack(const HeurTable &tb, const HeurLayout &L, uint8_t *in) {
    const InSlices s = in_slices(L);
    const whmec_problem *p = tb.p;
    std::memcpy(in + s.rc, tb.rc.data(), 4ull * L.n);
    std::memcpy(in + s.mc, tb.mc.data(), 4ull * L.n);
    float *ev = (float *)(in + s.ev);
    uint32_t *ent_col = (uint32_t *)(in + s.ent_col), *read_off = (uint32_t *)(in + s.read_off);
    const uint64_t base = p->read_off[0];
    for (uint64_t e = 0; e < L.nnz; ++e) {
        const int8_t a = (int8_t)p->ent_allele[base + e];
        const float q = (float)(int)p->ent_phred[base + e];
        ev[e] = q * a - q * (1 - a);  // heuristic.cpp's vote of an entry, same operands
        ent_col[e] = p->ent_col[base + e];
    }
    for (uint32_t r = 0; r <= L.m; ++r) read_off[r] = (uint32_t)(p->read_off[r] - base);
    std::memcpy(in + s.last, tb.last.data(), 4ull * L.m);
    std::memcpy(in + s.sample, tb.sample_of_read.data(), 4ull * L.m);
    std::memcpy(in + s.start, tb.start.data(), 4ull * (L.n + 1));
    int8_t *gt = (int8_t *)(in + s.gt);
    for (size_t i = 0; i < (size_t)L.S * L.n; ++i) gt[i] = (int8_t)tb.gt[i];
    if (L.n_trios) std::memcpy(in + s.trios, tb.trios.data(), 12ull * L.n_trios);
    std::memcpy(in + s.seen, tb.seen.data(), L.S);
}

HeurDevTable heur_bind(const HeurLayout &L, uint8_t *in, uint8_t *work, uint8_t *out) {
    const InSlices si = in_slices(L);
    const WorkSlices sw = work_slices(L);
    const OutSlices so = out_slices(L);
    uint8_t *i0 = in + L.in_off, *w0 = work + L.work_off, *o0 = out + L.out_off;
    HeurDevTable d;
    d.rc = (const float *)(i0 + si.rc);
    d.mc = (const float *)(i0 + si.mc);
    d.ev = (const float *)(i0 + si.ev);
    d.read_off = (const uint32_t *)(i0 + si.read_off);
    d.ent_col = (const uint32_t *)(i0 + si.ent_col);
    d.last = (const uint32_t *)(i0 + si.last);
    d.sample = (const uint32_t *)(i0 + si.sample);
    d.start = (const uint32_t *)(i0 + si.start);
    d.gt = (const int8_t *)(i0 + si.gt);
    d.trios = (const uint32_t *)(i0 + si.trios);
    d.seen = (const uint8_t *)(i0 + si.seen);
    for (int b = 0; b < 2; ++b) {
        d.rows[b].votes = (float *)(w0 + sw.votes[b]);
        d.rows[b].side = w0 + sw.side[b];
        d.rows[b].placed = w0 + sw.placed[b];
        d.rows[b].tv = (uint32_t *)(w0 + sw.tv[b]);
        d.rows[b].score = (float *)(w0 + sw.score[b]);
        d.rows[b].mut = (float *)(w0 + sw.mut[b]);
        d.rows[b].from = (uint32_t *)(w0 + sw.from[b]);
    }
    d.ht = (int32_t *)(w0 + sw.ht);
    d.a0 = (uint32_t *)(w0 + sw.a[0]);
    d.a1 = (uint32_t *)(w0 + sw.a[1]);
    d.a2 = (uint32_t *)(w0 + sw.a[2]);
    d.a3 = (uint32_t *)(w0 + sw.a[3]);
    d.best = (unsigned long long *)(w0 + sw.best);
    d.f0 = (float *)(w0 + sw.f0);
    d.f1 = (float *)(w0 + sw.f1);
    d.add = (float *)(w0 + sw.add);
    d.equal_to = (int32_t *)(w0 + sw.equal_to);
    d.active = (uint32_t *)(w0 + sw.active);
    d.kept = (uint32_t *)(w0 + sw.kept);
    d.back = (uint16_t *)(w0 + sw.back);
    d.rtv = (uint32_t *)(w0 + sw.rtv);
    d.rplaced = w0 + sw.rplaced;
    d.part = o0 + so.part;
    d.tv_out = (uint32_t *)(o0 + so.tv);
    d.status = (int32_t *)(o0 + so.status);
    d.n = L.n;
    d.m = L.m;
    d.S = L.S;
    d.n_trios = L.n_trios;
    d.row_limit = L.row_limit;
    d.cap = L.cap;
    d.rcap = L.rcap;
    d.Wmax = L.Wmax;
    d.Amax = L.Amax;
    d.NNmax = L.NNmax;
    d.ht_mask = L.ht_size - 1;
    d.distrust = L.distrust;
    return d;
}

const uint32_t *heur_out_tv(const HeurLayout &L, const uint8_t *out) { return (const uint32_t *)(out + L.out_off + out_slices(L).tv); }
int32_t heur_out_status(const HeurLayout &L, const uint8_t *out) {
    int32_t st;
    std::memcpy(&st, out + L.out_off + out_slices(L).status, 4);
    return st;
}

}  // namespace whmec

using namespace whmec;

extern "C" int whmec_heuristic_batch(const whmec_problem *const *problems, whmec_heuristic_solution *const *solutions, const uint32_t *row_limits,
                                     const int *allow_mutations, uint32_t n_tables, int device, int *status, char *errs, size_t errlen,
                                     whmec_stats *stats, whmec_stats *total) {
    if (n_tables == 0) return WHMEC_OK;
    if (!problems || !solutions || !row_limits || !allow_mutations || !status) return WHMEC_ERR_INPUT;
    for (uint32_t t = 0; t < n_tables; ++t)
        if (!problems[t] || !solutions[t]) return WHMEC_ERR_INPUT;
    if (stats) std::memset(stats, 0, sizeof(whmec_stats) * n_tables);
    if (total) std::memset(total, 0, sizeof(whmec_stats));
    auto fail_all = [&](int code, const std::string &msg) {
        for (uint32_t t = 0; t < n_tables; ++t) {
            status[t] = code;
            set_err(errs, errlen, t, msg);
        }
        return code;
    };
    auto host = [&](uint32_t t) {
        status[t] = whmec_heuristic(problems[t], row_limits[t], allow_mutations[t], solutions[t], errs ? errs + (size_t)t * errlen : nullptr,
                                    errs ? errlen : 0);
    };
    try {
        std::vector<HeurTable> tables(n_tables);
        std::vector<HeurLayout> layouts;
        std::vector<uint32_t> on_host;
        for (uint32_t t = 0; t < n_tables; ++t) {
            std::string msg;
            HeurTable &tb = tables[t];
            if (allow_mutations[t] == 0 || heur_prepare(tb, problems[t], true, solutions[t], msg) != WHMEC_OK || !heur_device_table(tb)) {
                on_host.push_back(t);  // (errors too: whmec_heuristic gives them with its own text and side effects)
                continue;
            }
            layouts.push_back(heur_layout(tb, std::min(row_limits[t], HEUR_MAX_ROWS)));
            layouts.back().table = t;
        }
        std::string msg;
        uint64_t budget = layouts.empty() ? 0 : heur_budget(device, msg);
        if (!msg.empty()) return fail_all(WHMEC_ERR_CUDA, msg);
        // WHMEC_HEURISTIC_ARENA_BUDGET=bytes (test hook): the bytes one group may take
        if (const char *e = std::getenv("WHMEC_HEURISTIC_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(e, nullptr, 10));
        std::vector<uint32_t> alone;
        const std::vector<HeurGroup> groups = layouts.empty() ? std::vector<HeurGroup>() : heur_groups(layouts, budget, alone);
        for (uint32_t i : alone) on_host.push_back(layouts[i].table);
        float ms_all = 0;
        uint64_t h2d = 0, d2h = 0;
        for (const HeurGroup &g : groups) {
            std::vector<uint8_t> in(g.in_bytes, 0), out;
            for (uint32_t i : g.members) heur_pack(tables[layouts[i].table], layouts[i], in.data() + layouts[i].in_off);
            float ms = 0;
            const int rc = heur_run_group(device, layouts, g, in, out, &ms, msg);
            if (rc != WHMEC_OK) return fail_all(rc, msg);
            ms_all += ms;
            h2d += g.in_bytes;
            d2h += g.out_bytes;
            for (uint32_t i : g.members) {
                const HeurLayout &L = layouts[i];
                const uint32_t t = L.table;
                if (heur_out_status(L, out.data()) != HEUR_OK) {
                    on_host.push_back(t);  // a row buffer overflowed: the host solver takes the table
                    continue;
                }
                heur_finish(tables[t], heur_out_part(L, out.data()), heur_out_tv(L, out.data()), solutions[t]);
                status[t] = WHMEC_OK;
                if (stats) {
                    stats[t].path_kind = 6;
                    stats[t].cells = L.work;
                    stats[t].max_active = L.Amax;
                    stats[t].transmissions = 1u << (2 * L.n_trios);
                }
            }
        }
        tables.clear();
        for (uint32_t t : on_host) host(t);
        if (total) {
            total->sweep_ms = ms_all;
            total->kernel_launches = (uint32_t)groups.size();
            total->h2d_bytes = h2d;
            total->d2h_bytes = d2h;
            total->path_kind = on_host.empty() && !groups.empty() ? 6 : 0;
        }
    } catch (const std::bad_alloc &) {
        return fail_all(WHMEC_ERR_UNSUPPORTED, "out of host memory");
    }
    return WHMEC_OK;
}
