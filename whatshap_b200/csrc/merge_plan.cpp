// Read merging of `whatshap phase --merge-reads` (whmec_merge_reads, DESIGN §4.17): validation, partners, chunk cuts, the removal
// loop and the output on the host, and the C entry point.  The rules restate ReadMerger.merge (whatshap/merge.py); the pair
// evaluation, the hooking and the sums are merge.h's, run by merge.cu.
#include "merge_plan.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <new>
#include <unordered_map>

namespace whmec {

namespace {

void put_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = '\0';
    }
}

uint32_t bits_for(uint64_t max_value) {  // bits that hold 0 .. max_value
    uint32_t b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return b;
}

std::string check(const whmec_merge_input *in, const whmec_merge_output *out) {
    if (!in || !out || !in->set_off || !out->out_off || (in->n_sets && (!out->error_kind || !out->error_read))) return "null arguments";
    const uint32_t ns = in->n_sets;
    if (in->set_off[0] != 0) return "set_off must start at 0";
    for (uint32_t s = 0; s < ns; ++s)
        if (in->set_off[s + 1] < in->set_off[s]) return "set_off must not decrease";
    const uint64_t nr = in->set_off[ns];
    if (!nr) return std::string();
    if (!in->read_off || !out->representative) return "null read arrays";
    if (in->read_off[0] != 0) return "read_off must start at 0";
    for (uint64_t r = 0; r < nr; ++r)
        if (in->read_off[r + 1] < in->read_off[r]) return "read_off must not decrease";
    if (in->read_off[nr] && (!in->position || !in->allele || !in->quality)) return "null entries";
    return std::string();
}

template <class T>
T *alloc_copy(const std::vector<T> &v) {
    T *p = (T *)std::malloc(std::max<size_t>(v.size(), 1) * sizeof(T));
    if (!p) throw std::bad_alloc();
    if (!v.empty()) std::memcpy(p, v.data(), v.size() * sizeof(T));
    return p;
}

double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// kill[j]: the first k > j with begin[k] >= end[j] (n if none).  Right to left, the stack holds the prefix-maximum records of
// begin[j + 1 ..], begins falling from bottom to top; the answer is the topmost record at or above end[j].
std::vector<uint32_t> first_kill(const std::vector<int64_t> &begin, const std::vector<uint64_t> &roff) {
    const uint32_t n = (uint32_t)begin.size();
    std::vector<uint32_t> kill(n), st;
    for (uint32_t j = n; j-- > 0;) {
        const int64_t end = begin[j] + (int64_t)(roff[j + 1] - roff[j]);
        size_t lo = 0, hi = st.size();  // records st[0 .. t) have begin >= end
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if (begin[st[mid]] >= end) lo = mid + 1;
            else hi = mid;
        }
        kill[j] = lo ? st[lo - 1] : n;
        while (!st.empty() && begin[st.back()] <= begin[j]) st.pop_back();
        st.push_back(j);
    }
    return kill;
}

struct Edge {
    uint32_t j, i;
    int64_t diff;
    bool notblue;
};

// networkx's bidirectional_shortest_path on the blue graph (adjacency in ascending neighbour id): expand the smaller fringe,
// forward on ties, return at the first meeting node.  Empty when v cannot be reached from u.
struct BiBfs {
    std::vector<uint32_t> pred_at, succ_at;  // epoch of the entry, 0 none
    std::vector<int64_t> pred, succ;         // -1 for the end itself
    uint32_t epoch = 0;

    std::vector<uint32_t> path(const std::vector<std::vector<uint32_t>> &adj, uint32_t u, uint32_t v) {
        if (pred_at.size() < adj.size()) pred_at.assign(adj.size(), 0), succ_at.assign(adj.size(), 0), pred.resize(adj.size()), succ.resize(adj.size());
        ++epoch;
        pred_at[u] = epoch, pred[u] = -1, succ_at[v] = epoch, succ[v] = -1;
        std::vector<uint32_t> fwd{u}, rev{v}, level;
        int64_t meet = -1;
        while (!fwd.empty() && !rev.empty() && meet < 0) {
            const bool forward = fwd.size() <= rev.size();
            std::vector<uint32_t> &fringe = forward ? fwd : rev;
            level.swap(fringe);
            fringe.clear();
            for (size_t a = 0; a < level.size() && meet < 0; ++a) {
                const uint32_t x = level[a];
                for (uint32_t w : adj[x]) {
                    if (forward) {
                        if (pred_at[w] != epoch) pred_at[w] = epoch, pred[w] = x, fringe.push_back(w);
                        if (succ_at[w] == epoch) { meet = w; break; }
                    } else {
                        if (succ_at[w] != epoch) succ_at[w] = epoch, succ[w] = x, fringe.push_back(w);
                        if (pred_at[w] == epoch) { meet = w; break; }
                    }
                }
            }
        }
        std::vector<uint32_t> p;
        if (meet < 0) return p;
        for (int64_t w = meet; w >= 0; w = pred[w]) p.push_back((uint32_t)w);
        std::reverse(p.begin(), p.end());
        for (int64_t w = succ[p.back()]; w >= 0; w = succ[w]) p.push_back((uint32_t)w);
        return p;
    }
};

uint64_t edge_key(uint32_t a, uint32_t b) { return a < b ? (uint64_t)a << 32 | b : (uint64_t)b << 32 | a; }

// The removal loop on the evaluated edges (blue, some also not-blue) and the roots of what is left.
void remove_and_join(MgCall &call, std::vector<Edge> &edges) {
    const uint32_t n = call.n_reads;
    std::vector<std::vector<uint32_t>> adj(n);
    std::unordered_map<uint64_t, int64_t> diff;
    diff.reserve(edges.size() * 2);
    std::vector<uint32_t> comp(n);
    for (uint32_t x = 0; x < n; ++x) comp[x] = x;
    for (const Edge &e : edges) {
        adj[e.j].push_back(e.i), adj[e.i].push_back(e.j);
        diff[edge_key(e.j, e.i)] = e.diff;
        mg_hook(comp.data(), e.j, e.i);
    }
    for (auto &a : adj) std::sort(a.begin(), a.end());
    for (uint32_t x = 0; x < n; ++x) comp[x] = mg_find(comp.data(), x);
    std::sort(edges.begin(), edges.end(), [](const Edge &a, const Edge &b) { return a.j != b.j ? a.j < b.j : a.i < b.i; });
    BiBfs bfs;
    for (const Edge &e : edges) {
        if (!e.notblue || comp[e.j] != comp[e.i]) continue;
        for (;;) {
            const std::vector<uint32_t> p = bfs.path(adj, e.j, e.i);
            if (p.empty()) break;
            size_t best = 0;
            int64_t best_d = diff[edge_key(p[0], p[1])];
            for (size_t k = 1; k + 1 < p.size(); ++k) {
                const int64_t d = diff[edge_key(p[k], p[k + 1])];
                if (d < best_d) best = k, best_d = d;
            }
            const uint32_t a = p[best], b = p[best + 1];
            adj[a].erase(std::find(adj[a].begin(), adj[a].end(), b));
            adj[b].erase(std::find(adj[b].begin(), adj[b].end(), a));
            ++call.st.removed_edges;
        }
    }
    call.parent.resize(n);
    for (uint32_t x = 0; x < n; ++x) call.parent[x] = x;
    for (uint32_t x = 0; x < n; ++x)
        for (uint32_t y : adj[x])
            if (x < y) mg_hook(call.parent.data(), x, y);
    for (uint32_t x = 0; x < n; ++x) call.parent[x] = mg_find(call.parent.data(), x);
}

struct Out {
    std::vector<uint64_t> read, entry_off{0};
    std::vector<int32_t> position;
    std::vector<uint8_t> allele;
    std::vector<int64_t> quality;
};

int run_set(const whmec_merge_input *in, uint32_t s, int device, uint64_t budget, MgCall &call, whmec_merge_output *out, Out &o,
            std::string &msg) {
    auto t0 = std::chrono::steady_clock::now();
    const uint64_t r0 = in->set_off[s], r1 = in->set_off[s + 1], n = r1 - r0;
    out->error_kind[s] = 0, out->error_read[s] = 0;
    if (n >= (1ull << 32) - 1) {
        msg = "whmec_merge_reads: a readset has 2^32 reads or more";
        return WHMEC_ERR_UNSUPPORTED;
    }
    const uint64_t e0 = n ? in->read_off[r0] : 0;
    // the first read that raises: an empty read (IndexError at read[0]) or an allele other than 0 or 1 (AssertionError)
    for (uint64_t r = r0; r < r1; ++r) {
        int kind = in->read_off[r + 1] == in->read_off[r] ? 1 : 0;
        for (uint64_t x = in->read_off[r]; x < in->read_off[r + 1] && !kind; ++x)
            if (in->allele[x] > 1) kind = 2;
        if (kind) {
            out->error_kind[s] = kind, out->error_read[s] = r - r0;
            for (uint64_t q = r0; q < r1; ++q) out->representative[q] = -1;
            call.st.plan_ms += (float)ms_since(t0);
            return WHMEC_OK;
        }
    }
    call.n_reads = (uint32_t)n;
    call.roff.resize(n + 1);
    call.begin.resize(n);
    call.woff.resize(n + 1);
    call.roff[0] = 0, call.woff[0] = 0;
    for (uint64_t r = 0; r < n; ++r) {
        call.roff[r + 1] = in->read_off[r0 + r + 1] - e0;
        call.begin[r] = in->position[in->read_off[r0 + r]];
        call.woff[r + 1] = call.woff[r] + (call.roff[r + 1] - call.roff[r] + 63) / 64;
    }
    call.n_entries = call.roff[n];
    call.allele = in->allele + e0;
    const std::vector<uint32_t> kill = first_kill(call.begin, call.roff);
    call.pstart.resize(n + 1);
    call.pstart[0] = 0;
    for (uint64_t j = 0; j < n; ++j) call.pstart[j + 1] = call.pstart[j] + (kill[j] - j - 1);
    const uint64_t np = call.pstart[n];
    call.st.reads += n, call.st.entries += call.n_entries, call.st.pairs += np;
    call.host_edges = (__int128)call.thr_diff + call.thr_neg_diff <= 0;
    const uint64_t fixed = n * MG_READ_BYTES + (call.woff[n] + 1) * MG_WORD_BYTES + call.n_entries + (1 << 20);
    const uint64_t cap = budget > fixed ? budget - fixed : 0;
    const uint64_t chunk_pairs = std::max<uint64_t>(1, std::min<uint64_t>(cap / MG_PAIR_BYTES, (1ull << 31) - 1));
    call.st.plan_ms += (float)ms_since(t0);
    int rc;
    if (n && (rc = mg_open_set(device, call, msg))) return rc;
    // the pairs, chunk after chunk; the blue edges are hooked on the device or come back for the removal loop
    std::vector<Edge> edges;
    call.blue = 0;
    for (uint64_t p0 = 0; p0 < np; p0 += chunk_pairs) {
        call.p0 = p0, call.p1 = std::min(np, p0 + chunk_pairs);
        ++call.st.chunks;
        if ((rc = mg_run_pairs(device, call, msg))) return rc;
        if (!call.host_edges) continue;
        t0 = std::chrono::steady_clock::now();
        uint32_t j = 0, i = 0;
        mg_pair(call.p0, call.pstart.data(), call.n_reads, j, i);
        for (uint64_t p = call.p0; p < call.p1; ++p, ++i) {
            while (call.pstart[j + 1] <= p) ++j, i = j + 1;
            const uint8_t f = call.flag[p - call.p0];
            if (f & MG_BLUE) edges.push_back(Edge{j, i, call.diff[p - call.p0], (f & MG_NOTBLUE) != 0});
        }
        call.st.plan_ms += (float)ms_since(t0);
    }
    if (call.host_edges) {
        t0 = std::chrono::steady_clock::now();
        call.st.blue_edges += edges.size();
        for (const Edge &e : edges) call.st.notblue_edges += e.notblue;
        remove_and_join(call, edges);
        call.st.plan_ms += (float)ms_since(t0);
    } else {
        call.st.blue_edges += call.blue;
        if (n && (rc = mg_roots(device, call, msg))) return rc;
    }
    t0 = std::chrono::steady_clock::now();
    // components of two reads or more, by representative, and their members' entries
    std::vector<uint64_t> size(n, 0), ent(n, 0);
    for (uint64_t r = 0; r < n; ++r) ++size[call.parent[r]], ent[call.parent[r]] += call.roff[r + 1] - call.roff[r];
    std::vector<uint32_t> reps, members, mstart(n + 1, 0);
    for (uint64_t r = 0; r < n; ++r) {
        out->representative[r0 + r] = call.parent[r];
        if (size[r] >= 2) reps.push_back((uint32_t)r);
        if (size[call.parent[r]] >= 2) ++mstart[call.parent[r] + 1];
    }
    for (uint64_t r = 0; r < n; ++r) mstart[r + 1] += mstart[r];
    members.resize(mstart[n]);
    {
        std::vector<uint32_t> fill(mstart.begin(), mstart.end() - 1);
        for (uint64_t r = 0; r < n; ++r)
            if (size[call.parent[r]] >= 2) members[fill[call.parent[r]]++] = (uint32_t)r;
    }
    call.st.merged_components += reps.size();
    // the merged reads' sums, whole components per chunk beside the resident set
    std::vector<uint64_t> run_off(reps.size() + 1, 0);
    std::vector<MgRun> runs;
    call.st.plan_ms += (float)ms_since(t0);
    for (size_t c0 = 0; c0 < reps.size();) {
        t0 = std::chrono::steady_clock::now();
        size_t c1 = c0;
        uint64_t ne = 0;
        while (c1 < reps.size()) {
            const uint64_t e = ent[reps[c1]];
            if (c1 > c0 && ((ne + e) * MG_ENTRY_BYTES > cap || ne + e >= (1ull << 31))) break;
            ne += e, ++c1;
        }
        if (ne >= (1ull << 31)) {
            msg = "whmec_merge_reads: a merged read has 2^31 entries or more";
            return WHMEC_ERR_UNSUPPORTED;
        }
        call.entries.clear();
        int32_t pmin = INT32_MAX, pmax = INT32_MIN;
        for (size_t c = c0; c < c1; ++c)
            for (uint32_t k = mstart[reps[c]]; k < mstart[reps[c] + 1]; ++k) {
                const uint64_t r = members[k];
                for (uint64_t x = in->read_off[r0 + r]; x < in->read_off[r0 + r + 1]; ++x) {
                    call.entries.push_back(MgEntry{(uint32_t)(c - c0), in->position[x], in->quality[x], in->allele[x]});
                    pmin = std::min(pmin, in->position[x]), pmax = std::max(pmax, in->position[x]);
                }
            }
        call.n_comp = (uint32_t)(c1 - c0);
        call.pmin = pmin;
        call.pos_bits = bits_for((uint64_t)((int64_t)pmax - pmin));
        ++call.st.chunks;
        call.st.plan_ms += (float)ms_since(t0);
        if ((rc = mg_run_accumulate(device, call, msg))) return rc;
        for (const MgRun &run : call.runs) ++run_off[c0 + run.comp + 1];
        runs.insert(runs.end(), call.runs.begin(), call.runs.end());
        c0 = c1;
    }
    t0 = std::chrono::steady_clock::now();
    for (size_t c = 0; c < reps.size(); ++c) run_off[c + 1] += run_off[c];
    // the output: singletons as they came, representatives with their sums, other members dropped
    for (uint64_t r = 0, c = 0; r < n; ++r) {
        const uint32_t root = call.parent[r];
        if (size[root] >= 2 && root != r) continue;
        o.read.push_back(r);
        if (size[root] >= 2) {
            for (uint64_t k = run_off[c]; k < run_off[c + 1]; ++k)
                o.position.push_back(runs[k].pos), o.allele.push_back((uint8_t)runs[k].allele), o.quality.push_back(runs[k].quality);
            ++c;
        } else {
            for (uint64_t x = in->read_off[r0 + r]; x < in->read_off[r0 + r + 1]; ++x)
                o.position.push_back(in->position[x]), o.allele.push_back(in->allele[x]), o.quality.push_back(in->quality[x]);
        }
        o.entry_off.push_back(o.position.size());
    }
    call.st.plan_ms += (float)ms_since(t0);
    return WHMEC_OK;
}

}  // namespace

}  // namespace whmec

using namespace whmec;

extern "C" void whmec_merge_reads_release(whmec_merge_output *out) {
    if (!out) return;
    for (void *p : {(void *)out->out_read, (void *)out->out_entry_off, (void *)out->out_position, (void *)out->out_allele,
                    (void *)out->out_quality})
        std::free(p);
    out->out_read = out->out_entry_off = nullptr;
    out->out_position = nullptr, out->out_allele = nullptr, out->out_quality = nullptr, out->n_out = 0;
}

extern "C" int whmec_merge_reads(const whmec_merge_input *in, int device, whmec_merge_output *out, whmec_merge_stats *stats, char *err,
                                 size_t errlen) {
    const std::string bad = check(in, out);
    if (!bad.empty()) {
        put_err(err, errlen, "whmec_merge_reads: " + bad);
        return WHMEC_ERR_INPUT;
    }
    out->n_out = 0;
    out->out_read = out->out_entry_off = nullptr;
    out->out_position = nullptr, out->out_allele = nullptr, out->out_quality = nullptr;
    std::string msg;
    const uint64_t budget = mg_budget(device, msg);
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    MgCall call;
    call.thr_diff = in->thr_diff, call.thr_neg_diff = in->thr_neg_diff, call.max_error_rate = in->max_error_rate;
    try {
        Out o;
        out->out_off[0] = 0;
        for (uint32_t s = 0; s < in->n_sets; ++s) {
            const int rc = run_set(in, s, device, budget, call, out, o, msg);
            if (rc != WHMEC_OK) {
                mg_close(call);
                put_err(err, errlen, msg);
                return rc;
            }
            out->out_off[s + 1] = o.read.size();
        }
        mg_close(call);
        call.st.output_reads = o.read.size();
        out->n_out = o.read.size();
        out->out_read = alloc_copy(o.read), out->out_entry_off = alloc_copy(o.entry_off);
        out->out_position = alloc_copy(o.position), out->out_allele = alloc_copy(o.allele), out->out_quality = alloc_copy(o.quality);
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        mg_close(call);
        whmec_merge_reads_release(out);
        put_err(err, errlen, "whmec_merge_reads: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    } catch (const std::exception &e) {  // nothing may cross the C boundary
        mg_close(call);
        whmec_merge_reads_release(out);
        put_err(err, errlen, std::string("whmec_merge_reads: ") + e.what());
        return WHMEC_ERR_UNSUPPORTED;
    }
}
