// Host side of the sinc resampler (resample.cu) behind fac_resample* / fac_rs_pool_*: filter tables per rate pair and
// pools of resampler sessions, held by a handle through one RsHost.
#pragma once
#include <cuda_runtime.h>
#include <string>

#include "../../include/facodec_b200.h"

namespace fac {

struct RsHost;

// What the resampler needs of a handle: its device, its error text, its launch counter and its RsHost (created on use).
struct RsEnv {
    int device;
    std::string& err;
    int& launches;
    RsHost*& host;
};

// Reduced geometry of a rate pair: out4 = {orig, new, width, K}.  FAC_ERR_INVALID for an unsupported pair.
int rs_geometry(int orig, int nw, int* out4);
long long rs_out_len(int orig, int nw, long long n);
long long rs_ready(int orig, int nw, int quantum, long long seen, long long emitted);

int rs_table(RsEnv e, int orig, int nw, const float* table_host);
int rs_resample(RsEnv e, const float* x, int B, int T, const int* lengths, int orig, int nw, float* y, cudaStream_t st);
int rs_pool_create(RsEnv e, int capacity, int quantum);
int rs_pool_open(RsEnv e, int pool_id, int orig, int nw);
int rs_pool_step(RsEnv e, int pool_id, int n, const int* sessions, const int* T, const float* const* x, float* const* y,
                 int* counts, bool finish, cudaStream_t st);
int rs_pool_undo(RsEnv e, int pool_id, int n, const int* sessions);
int rs_pool_close(RsEnv e, int pool_id, int session);
int rs_pool_destroy(RsEnv e, int pool_id);
void rs_host_free(RsHost* host);

// One pool session's state as fac_*_pool_export / _import move it (engine.cu): the header's counters and the slot's device
// regions, in payload order.
struct SlotState {
    long long counters[FAC_STATE_COUNTERS] = {};
    void* region[FAC_STATE_REGIONS] = {};
    long long bytes[FAC_STATE_REGIONS] = {};
    int nreg = 0;
};
// The state of open session `session` of a resampler pool (FAC_ERR_STATE once finished).
int rs_slot_read(RsEnv e, int pool_id, int session, SlotState& s, const char* who);
// Checks an imported state's counters and region sizes against the pool and the pair's table, and readies a free slot for
// it (its buffers grown if need be): s.region[0] becomes the slot's history buffer.  Returns the slot or a status; nothing
// an open session sees changes.
int rs_slot_place(RsEnv e, int pool_id, SlotState& s, const char* who);
// Opens the slot rs_slot_place readied, with the state's counters (no step to take back).
void rs_slot_commit(RsEnv e, int pool_id, int slot, const SlotState& s);

}  // namespace fac
