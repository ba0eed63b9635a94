// Tile kernel path (T == 1): declared here, defined in tile.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "pack.h"
#include "tile_plan.h"

namespace whmec {

// free device memory plus what the stream-ordered pool holds but does not use
size_t device_available_bytes();

struct TilePlan {
    uint64_t backptr_bytes = 0;
    uint64_t state_bytes = 0;     // projection state moved through global memory by one sweep
    uint32_t launches = 0;
    std::string why;              // reason when plan() returns false
    bool over_hbm = false;        // create() refused: state + back-pointers exceed the free HBM
    void *impl = nullptr;
    // Host-only: decide whether the tile path applies and build its schedule.
    bool plan(const Packed &pk);
    // Host-only: take over a schedule planned elsewhere (the union of several tables' schedules, tile_plan.h: merge_tile_tables).
    void adopt(TileSchedule &&ts);
    // `d_cols`: the packer's per-column records on the device (uploaded by the caller while the host planned; owned by the caller)
    int create(const Packed &pk, cudaStream_t stream, uint64_t &h2d_bytes, std::string &msg, const ColMeta *d_cols);
    int sweep(const Packed &pk, cudaStream_t stream, std::string &msg);
    int backtrace(const Packed &pk, cudaStream_t stream, uint32_t *d_path_index, uint32_t *d_result, std::string &msg);
    // Several tables in one sweep: costs[t] = sum of the optima of the chains [table_chain[t], table_chain[t + 1]) (device pointers).
    int table_costs(cudaStream_t stream, const uint32_t *d_table_chain, uint32_t n_tables, uint32_t *d_costs, std::string &msg);
    void release(cudaStream_t stream);
};

}  // namespace whmec
