// K-mer pair counts of `whatshap learn` (whmec_learn, DESIGN §4.13): the host walk, floors, variant windows, chunk cut and the C
// entry points.  The walk restates Caller::enumerate_kmers (src/caller.cpp) once per alignment at O(CIGAR operations); the
// device work of a chunk is ln_run_chunk (learn.cu).
#include "learn_plan.h"

#include <algorithm>
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

namespace whmec {

namespace {

void put_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = '\0';
    }
}

struct LnWalk {
    uint64_t kmers = 0;
    int64_t first = 0, last = 0;  // columns of the first and last k-mer
};

// enumerate_kmers of alignment a as runs (written to ops, n_ops of them); empty, or the reason the reference aborts or reads out
// of bounds.
std::string walk(const whmec_learn_input &in, uint32_t a, LnOp *ops, uint32_t &n_ops, LnWalk &w) {
    const uint64_t c0 = in.cigar_off[a], nc = in.cigar_off[a + 1] - c0, qlen = in.query_off[a + 1] - in.query_off[a];
    const int64_t k = in.k, L = (int64_t)in.reference_len;
    if (qlen >= (1ull << 31)) return "the query is longer than 2^31 - 1";
    int64_t pos = in.reference_start[a];
    uint64_t ci = 0, i = 0;
    uint32_t reset = 0;
    n_ops = 0;
    uint8_t op = nc ? in.cigar_op[c0] : 0;
    int64_t len = nc ? in.cigar_len[c0] : 0;
    if (qlen && !nc) return "the CIGAR ends while query bytes remain";
    while (i < qlen) {
        for (;;) {  // the operations that consume no query byte
            if (op == 2 || op == 3) pos += len;
            else if (op == 4) reset = (uint32_t)i;
            else if (len != 0 && op != 5) break;
            if (++ci >= nc) return "the CIGAR ends while query bytes remain";
            op = in.cigar_op[c0 + ci];
            len = in.cigar_len[c0 + ci];
        }
        if (op != 0 && op != 1 && op != 7 && op != 8)
            return "CIGAR operation " + std::to_string(op) + " of length " + std::to_string(len) + " while query bytes remain (the reference asserts)";
        const uint64_t take = std::min<uint64_t>((uint64_t)len, qlen - i);
        const bool adv = op != 1;
        if (pos < INT32_MIN || pos + (int64_t)take + 1 > INT32_MAX) return "a reference position outside int32";
        const LnOp o{(uint32_t)i, (uint32_t)take, reset, (int32_t)(pos + 1), adv ? 1u : 0u};
        ops[n_ops++] = o;
        const uint64_t e0 = std::max<uint64_t>(i, (uint64_t)reset + k - 1), e1 = i + take;
        if (e0 < e1) {
            if (!w.kmers) w.first = ln_col(o, (uint32_t)e0);
            w.last = ln_col(o, (uint32_t)(e1 - 1));
            w.kmers += e1 - e0;
        }
        if (adv) pos += take;
        i += take;
        len -= take;
    }
    if (!w.kmers) return "the query has no k-mer (the reference reads an empty list)";
    if (in.reference_start[a] + k - 1 > L) return "pos + k - 1 lies beyond the reference (the reference reads past its k-mers)";
    if (w.last > L) return "a k-mer column lies beyond the reference (the reference reads past its k-mers)";
    return std::string();
}

// The kept k-mers of read r in columns [lo, hi] run by run: fn(run, first byte, end byte, first column, last column).
template <class F>
void kept_runs(const LnRead &r, const LnOp *ops, uint32_t k, int64_t lo, int64_t hi, F &&fn) {
    lo = std::max<int64_t>(lo, (int64_t)r.floor + 1);
    for (uint32_t j = 0; j < r.n_ops; ++j) {
        const LnOp &o = ops[r.op0 + j];
        int64_t e0 = std::max<int64_t>(o.q0, (int64_t)o.reset + k - 1), e1 = (int64_t)o.q0 + o.len;
        if (e0 >= e1) continue;
        if (o.adv) {
            e0 = std::max<int64_t>(e0, o.q0 + (lo - o.col0));
            e1 = std::min<int64_t>(e1, o.q0 + (hi - o.col0) + 1);
            if (e0 >= e1) continue;
        } else if (o.col0 < lo || o.col0 > hi) {
            continue;
        }
        fn(o, (uint32_t)e0, (uint32_t)e1, ln_col(o, (uint32_t)e0), ln_col(o, (uint32_t)(e1 - 1)));
    }
}

}  // namespace

uint32_t ln_intervals(const int32_t *pos, const int32_t *len, uint32_t n, uint32_t off, int64_t lo, int64_t hi, int64_t window,
                      int64_t k, std::vector<int64_t> &iv) {
    int64_t c = lo;
    while (c <= hi) {
        const int64_t s0 = (int64_t)pos[off] - window, s1 = (int64_t)pos[off] + len[off] - 1 + window + k - 1;
        const bool next = off + 1 < n;
        const int64_t n0 = next ? (int64_t)pos[off + 1] - window : 0, n1 = next ? (int64_t)pos[off + 1] + len[off + 1] - 1 + window : -1;
        if (s0 <= c && c <= s1) {  // inside the front variant's window
            c = s1 + 1;
            continue;
        }
        if (next && n0 <= c && c <= n1) {  // inside the next one's: the front is popped, the column skipped
            ++off;
            ++c;
            continue;
        }
        int64_t e = hi;
        if (s0 > c) e = std::min(e, s0 - 1);
        if (next && n0 > c) e = std::min(e, n0 - 1);
        if (!iv.empty() && iv.back() + 1 == c) iv.back() = e;
        else iv.push_back(c), iv.push_back(e);
        c = e + 1;
    }
    return off;
}

std::vector<LnChunk> ln_chunks(LnCall &call, int64_t lo, int64_t hi, uint64_t cap) {
    std::vector<LnChunk> chunks;
    call.entries.clear();
    if (hi < lo) return chunks;
    // keys per column as a step function: a run of M, = or X adds `weight` keys per column over its kept columns, a run of I its
    // kept keys at one column
    struct Ev {
        int64_t col;
        int64_t slope;
        uint64_t mass;
    };
    std::vector<Ev> ev;
    std::vector<int64_t> span_lo(call.n_reads, INT64_MAX), span_hi(call.n_reads, INT64_MIN);
    for (uint32_t r = 0; r < call.n_reads; ++r) {
        const LnRead &rd = call.reads[r];
        kept_runs(rd, call.ops, call.k, lo, hi, [&](const LnOp &o, uint32_t e0, uint32_t e1, int64_t c0, int64_t c1) {
            if (o.adv) {
                ev.push_back(Ev{c0, (int64_t)rd.weight, 0});
                ev.push_back(Ev{c1 + 1, -(int64_t)rd.weight, 0});
            } else {
                ev.push_back(Ev{c0, 0, (uint64_t)(e1 - e0) * rd.weight});
            }
            span_lo[r] = std::min(span_lo[r], c0);
            span_hi[r] = std::max(span_hi[r], c1);
        });
    }
    std::sort(ev.begin(), ev.end(), [](const Ev &a, const Ev &b) { return a.col < b.col; });
    int64_t cur = lo, x = lo;
    uint64_t acc = 0, slope = 0;
    size_t e = 0;
    auto close = [&](int64_t end) {
        LnChunk c;
        c.lo = cur, c.hi = end;
        chunks.push_back(c);
        cur = end + 1;
        acc = 0;
    };
    auto add = [&](int64_t x0, int64_t n, uint64_t per_col) {  // columns x0 .. x0 + n - 1 with per_col keys each
        while (n > 0) {
            const uint64_t room = acc < cap ? cap - acc : 0;
            uint64_t fit = per_col ? room / per_col : (uint64_t)n;
            if (!fit) {
                if (x0 > cur) {
                    close(x0 - 1);
                    continue;
                }
                fit = 1;
            }
            const int64_t take = (int64_t)std::min<uint64_t>((uint64_t)n, fit);
            acc += (uint64_t)take * per_col;
            x0 += take;
            n -= take;
        }
    };
    while (x <= hi) {
        uint64_t mass = 0;
        for (; e < ev.size() && ev[e].col == x; ++e) slope += ev[e].slope, mass += ev[e].mass;
        add(x, 1, slope + mass);
        const int64_t nx = e < ev.size() ? std::min(ev[e].col, hi + 1) : hi + 1;
        if (nx > x + 1) add(x + 1, nx - x - 1, slope);
        x = nx;
    }
    if (cur <= hi) close(hi);
    // each chunk's entries: the reads whose kept columns meet it, in order of their first kept column
    std::vector<uint32_t> order;
    for (uint32_t r = 0; r < call.n_reads; ++r)
        if (span_lo[r] <= span_hi[r]) order.push_back(r);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return span_lo[a] < span_lo[b]; });
    std::vector<uint32_t> active;
    size_t p = 0;
    for (LnChunk &c : chunks) {
        for (; p < order.size() && span_lo[order[p]] <= c.hi; ++p) active.push_back(order[p]);
        active.erase(std::remove_if(active.begin(), active.end(), [&](uint32_t r) { return span_hi[r] < c.lo; }), active.end());
        c.e0 = (uint32_t)call.entries.size();
        for (uint32_t r : active) {
            const LnRead &rd = call.reads[r];
            LnEntry en{r, UINT32_MAX, 0, 0, c.n_keys};  // n_keys below
            uint64_t n = 0;
            kept_runs(rd, call.ops, call.k, c.lo, c.hi, [&](const LnOp &, uint32_t e0, uint32_t e1, int64_t, int64_t) {
                en.b0 = std::min(en.b0, e0);
                en.b1 = std::max(en.b1, e1);
                n += (uint64_t)(e1 - e0) * rd.weight;
            });
            if (!n) continue;
            en.n_keys = (uint32_t)n;  // < 2^32: a read has fewer than 2^31 bytes, each at most two keys
            call.entries.push_back(en);
            c.n_keys += n;
        }
        c.e1 = (uint32_t)call.entries.size();
        uint32_t bits = 2 * call.k;
        while (bits < 64 && (uint64_t)(c.hi - c.lo) >> (bits - 2 * call.k)) ++bits;
        c.wide = bits > 32;
    }
    return chunks;
}

}  // namespace whmec

using namespace whmec;

extern "C" int whmec_learn(const whmec_learn_input *in, int device, whmec_learn_output *out, whmec_learn_stats *stats, char *err,
                           size_t errlen) {
    if (!in || !out || (in->reference_len && !in->reference) ||
        (in->n_alignments && (!in->reference_start || !in->cigar_off || !in->query_off)) ||
        (in->n_alignments && in->cigar_off[in->n_alignments] && (!in->cigar_op || !in->cigar_len)) ||
        (in->n_alignments && in->query_off[in->n_alignments] && !in->query) || (in->n_variants && (!in->variant_pos || !in->variant_len))) {
        put_err(err, errlen, "whmec_learn: null or malformed arguments");
        return WHMEC_ERR_INPUT;
    }
    std::memset(out, 0, sizeof(*out));
    const int64_t k = in->k, L = (int64_t)in->reference_len;
    std::string bad;
    if (k < 1 || k > 15) bad = "whmec_learn: k must lie in 1..15";
    else if (in->reference_len >= (1ull << 31)) bad = "whmec_learn: the reference is longer than 2^31 - 1";
    else if (L < k) bad = "whmec_learn: the reference is shorter than k";
    else if (!in->n_variants) bad = "whmec_learn: the variant list is empty (the reference reads its front)";
    else if (in->first_variant >= in->n_variants) bad = "whmec_learn: first_variant lies beyond the variant list";
    for (uint64_t c = 0; bad.empty() && in->n_alignments && c < in->cigar_off[in->n_alignments]; ++c)
        if (in->cigar_len[c] < 0) bad = "whmec_learn: a negative CIGAR length";
    for (uint32_t a = 0; bad.empty() && in->floor && a < in->n_alignments; ++a)
        if (in->floor[a] < k - 1) bad = "whmec_learn: a floor below k - 1";
    if (!bad.empty()) {
        put_err(err, errlen, bad);
        return WHMEC_ERR_INPUT;
    }
    std::string msg;
    const uint64_t budget = ln_budget(device, msg);  // (first: selects the device and the page-locked staging memory)
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    LnCall call;
    try {
        const auto t0 = std::chrono::steady_clock::now();
        const uint32_t n = in->n_alignments;
        const uint64_t n_cigar = n ? in->cigar_off[n] : 0;
        StagedVec<LnOp> ops(std::max<uint64_t>(n_cigar, 1));
        StagedVec<LnRead> reads(std::max<uint32_t>(n, 1));
        std::vector<LnWalk> walks(n);
        const uint32_t threads = host_threads(32);
        const uint32_t n_tasks = std::max(1u, std::min(n, threads * 8));
        std::vector<std::string> errs(n_tasks);
        std::vector<uint32_t> err_at(n_tasks, UINT32_MAX);
        parallel_tasks(n_tasks, threads, [&](uint32_t t) {
            const uint32_t a0 = (uint32_t)((uint64_t)n * t / n_tasks), a1 = (uint32_t)((uint64_t)n * (t + 1) / n_tasks);
            for (uint32_t a = a0; a < a1; ++a) {
                uint32_t n_ops = 0;
                std::string e = walk(*in, a, ops.data() + in->cigar_off[a], n_ops, walks[a]);
                if (!e.empty()) {
                    errs[t] = "alignment " + std::to_string(a) + ": " + e;
                    err_at[t] = a;
                    return;
                }
                reads[a] = LnRead{in->query_off[a], in->cigar_off[a], n_ops, walks[a].kmers == 1 ? 2u : 1u, 0, 0};
            }
        });
        for (uint32_t t = 0; t < n_tasks; ++t)
            if (err_at[t] != UINT32_MAX) {  // the first failing alignment in input order
                put_err(err, errlen, errs[t]);
                return WHMEC_ERR_INPUT;
            }
        if (in->col_lo > 0 && (in->col_lo < k || in->col_hi > L)) {  // (after the walk, which names a read beyond L)
            put_err(err, errlen, "whmec_learn: the column range lies outside k..L");
            return WHMEC_ERR_INPUT;
        }
        int64_t top = k - 1;  // T: the last popped column after each add_read
        for (uint32_t a = 0; a < n; ++a) {
            reads[a].floor = in->floor ? in->floor[a] : (int32_t)top;
            top = std::max<int64_t>(top, (int64_t)in->reference_start[a] + k - 1);
            call.st.kmers += walks[a].kmers;
        }
        const int64_t lo = in->col_lo > 0 ? in->col_lo : k, hi = in->col_lo > 0 ? in->col_hi : in->final ? L : top;
        out->next_variant = ln_intervals(in->variant_pos, in->variant_len, in->n_variants, in->first_variant, lo, hi, in->window, k, call.iv);
        call.k = (uint32_t)k;
        call.query = in->query;
        call.query_bytes = n ? in->query_off[n] : 0;
        call.reads = reads.data();
        call.n_reads = n;
        call.ops = ops.data();
        call.n_ops = n_cigar;
        call.st.alignments = n;
        if (hi >= lo) {  // the reference's bytes b0 .. hi - 1, after the last k ACGT bytes before b0
            const int64_t b0 = lo - 1, nb = hi - b0;
            call.b0 = b0;
            std::vector<uint8_t> seed;
            for (int64_t j = b0 - 1; j >= 0 && (int64_t)seed.size() < k; --j)
                if (ln_code(in->reference[j]) < 4) seed.push_back((uint8_t)ln_code(in->reference[j]));
            call.code.assign(k - seed.size(), 0);
            call.code.insert(call.code.end(), seed.rbegin(), seed.rend());
            call.base.assign(nb / 32 + 1, 0);
            call.mask.assign(nb / 32 + 1, 0);
            for (int64_t x = 0; x < nb; ++x) {
                if (x % 32 == 0) call.base[x / 32] = (uint32_t)call.code.size();
                const uint32_t c = ln_code(in->reference[b0 + x]);
                if (c < 4) call.code.push_back((uint8_t)c), call.mask[x / 32] |= 1u << (x % 32);
            }
            if (nb % 32 == 0) call.base[nb / 32] = (uint32_t)call.code.size();
        }
        const uint64_t fixed = call.query_bytes + n_cigar * sizeof(LnOp) + (uint64_t)n * sizeof(LnRead) + call.code.size() +
                               call.base.size() * 8 + call.iv.size() * 8 + 16 * 256;  // (+ the 256-byte alignment of the arena's arrays)
        const uint64_t cap = std::min<uint64_t>((budget > fixed ? budget - fixed : 0) / LN_KEY_BYTES, 1ull << 30);
        const std::vector<LnChunk> chunks = ln_chunks(call, lo, hi, cap);
        call.st.plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        int rc = WHMEC_OK;
        for (const LnChunk &c : chunks) {
            if (!c.n_keys) continue;
            call.st.kept += c.n_keys;
            ++call.st.chunks;
            if ((rc = ln_run_chunk(device, call, c, msg)) != WHMEC_OK) break;
        }
        ln_close(call);
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        out->n_rows = call.rows.size() / 4;
        call.st.rows = out->n_rows;
        out->rows = (int32_t *)std::malloc(std::max<size_t>(call.rows.size(), 1) * sizeof(int32_t));
        if (!out->rows) throw std::bad_alloc();
        std::memcpy(out->rows, call.rows.data(), call.rows.size() * sizeof(int32_t));
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        ln_close(call);
        whmec_learn_release(out);
        put_err(err, errlen, "whmec_learn: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    } catch (const std::exception &e) {  // nothing may cross the C boundary
        ln_close(call);
        whmec_learn_release(out);
        put_err(err, errlen, std::string("whmec_learn: ") + e.what());
        return WHMEC_ERR_UNSUPPORTED;
    }
}

extern "C" void whmec_learn_release(whmec_learn_output *out) {
    if (!out) return;
    std::free(out->rows);
    out->rows = nullptr;
    out->n_rows = 0;
}

namespace {

char *put_int(char *p, int32_t v) {
    char tmp[12];
    int n = 0;
    uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    do tmp[n++] = (char)('0' + u % 10);
    while (u /= 10);
    if (v < 0) *p++ = '-';
    while (n) *p++ = tmp[--n];
    return p;
}

}  // namespace

extern "C" int whmec_learn_write(const char *path, const whmec_learn_output *out, int append, char *err, size_t errlen) {
    if (!path || !out || (out->n_rows && !out->rows)) {
        put_err(err, errlen, "whmec_learn_write: null arguments");
        return WHMEC_ERR_INPUT;
    }
    std::vector<char> buf;
    try {
        buf.resize(1 << 20);
    } catch (const std::bad_alloc &) {
        put_err(err, errlen, "whmec_learn_write: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    }
    FILE *f = std::fopen(path, append ? "ab" : "wb");
    if (!f) {
        put_err(err, errlen, std::string("whmec_learn_write: cannot open ") + path + ": " + std::strerror(errno));
        return WHMEC_ERR_INPUT;
    }
    char *p = buf.data();
    bool ok = true;
    for (uint64_t r = 0; r < out->n_rows && ok; ++r) {
        const int32_t *row = out->rows + 4 * r;
        for (int j = 0; j < 4; ++j) {
            p = put_int(p, row[j]);
            *p++ = j == 3 ? '\n' : '\t';
        }
        if (p - buf.data() > (ptrdiff_t)buf.size() - 64) {
            ok = std::fwrite(buf.data(), 1, p - buf.data(), f) == (size_t)(p - buf.data());
            p = buf.data();
        }
    }
    if (ok && p > buf.data()) ok = std::fwrite(buf.data(), 1, p - buf.data(), f) == (size_t)(p - buf.data());
    ok = (std::fclose(f) == 0) && ok;
    if (!ok) {
        put_err(err, errlen, std::string("whmec_learn_write: writing ") + path + " failed");
        return WHMEC_ERR_INPUT;
    }
    return WHMEC_OK;
}
