// Many heuristic tables in one call (whmec_heuristic_batch, DESIGN §4.10): the host plan.  Every table the device sweeps gets
// its own slices of one group arena (inputs, rows and records, outputs); heur_sweep (heuristic_device.h) runs on the slices.
// Plain C++ (used by heuristic_batch.cpp and by the test-only emulation, tests/emul/emul_heuristic_batch.cpp).
#pragma once
#include <string>
#include <vector>

#include "heuristic.h"
#include "heuristic_device.h"

namespace whmec {

constexpr uint32_t HEUR_THREADS = 256;  // threads of the CTA that sweeps one table

// One table of a group: its sizes, and where its slices start in the group's input, work and output regions (bytes).
struct HeurLayout {
    uint32_t table = 0;  // position in the caller's list
    uint32_t n = 0, m = 0, S = 0, n_trios = 0, row_limit = 0, distrust = 0;
    uint32_t cap = 0;    // rows per row buffer: 2 x row_limit x (2 for one individual, 4 for pedigrees), at least 64
    uint32_t rcap = 0;   // rows a column may record: 2 x row_limit, at least 64
    uint32_t Wmax = 0;   // widest vote window
    uint32_t Amax = 0;   // most reads active in one column (its new reads included)
    uint32_t NNmax = 0;  // most reads starting in one column
    uint32_t ht_size = 0;
    uint64_t nnz = 0;
    uint64_t in_bytes = 0, work_bytes = 0, out_bytes = 0;
    uint64_t in_off = 0, work_off = 0, out_off = 0;
    uint64_t work = 0;   // sum over columns of row_limit: the order in which tables are handed out, longest first
};

// A group: tables that share one arena and one launch.
struct HeurGroup {
    std::vector<uint32_t> members;  // positions in the layout list
    uint64_t in_bytes = 0, work_bytes = 0, out_bytes = 0;
};

// Whether a prepared table (heur_prepare, allow_mutations) can run on the device; false: whmec_heuristic runs it.
bool heur_device_table(const HeurTable &tb);
// The sizes of a prepared table under `row_limit` (already capped at 65535).
HeurLayout heur_layout(const HeurTable &tb, uint32_t row_limit);
// Tables in work order (longest first, list order on ties) cut into groups whose bytes stay within `budget`; a table that does
// not fit alone is listed in `alone`.  Sets every member's offsets.
std::vector<HeurGroup> heur_groups(std::vector<HeurLayout> &layouts, uint64_t budget, std::vector<uint32_t> &alone);
// The input slice of a table (host image at `in`, L.in_bytes long).
void heur_pack(const HeurTable &tb, const HeurLayout &L, uint8_t *in);
// The table's view of a group whose regions start at `in`, `work` and `out` (device or host addresses).
HeurDevTable heur_bind(const HeurLayout &L, uint8_t *in, uint8_t *work, uint8_t *out);
// The part of a table's output slice the host reads: partition [m], transmission [n], status.
inline const uint8_t *heur_out_part(const HeurLayout &L, const uint8_t *out) { return out + L.out_off; }
const uint32_t *heur_out_tv(const HeurLayout &L, const uint8_t *out);
int32_t heur_out_status(const HeurLayout &L, const uint8_t *out);

// Implemented by heuristic.cu (and by the emulation): the device bytes a group may take, and one group's run: upload of the
// descriptors and inputs, one launch, download of the output region into `out`.  ms: device time of the launch.
uint64_t heur_budget(int device, std::string &msg);
int heur_run_group(int device, const std::vector<HeurLayout> &layouts, const HeurGroup &g, std::vector<uint8_t> &in, std::vector<uint8_t> &out,
                   float *ms, std::string &msg);

}  // namespace whmec
