// Host side of the sinc resampler (resample.cu) behind fac_resample* / fac_rs_pool_*: filter tables per rate pair and
// pools of resampler sessions, held by a handle through one RsHost.
#pragma once
#include <cuda_runtime.h>
#include <string>

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

}  // namespace fac
