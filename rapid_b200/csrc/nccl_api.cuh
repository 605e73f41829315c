// NCCL through dlopen, shared by the sharded fast-round tally (fast_paxos.cu) and the sharded classic-Paxos tallies
// (classic_paxos.cu).  The library is loaded on first use; no NCCL header or link-time dependency is needed.
#pragma once

#include "common.cuh"

namespace rapid {

typedef struct { char internal[128]; } nccl_uid;
typedef void* nccl_comm;
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(nccl_uid*) = nullptr;
    int (*CommInitRank)(nccl_comm*, int, nccl_uid, int) = nullptr;
    int (*CommDestroy)(nccl_comm) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
    // optional: only the sharded classic-Paxos tallies need them, and they refuse with RAPID_ENCCL where they are missing
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
extern NcclApi g_nccl;
static const int NCCL_UINT8 = 1, NCCL_INT32 = 2, NCCL_UINT64 = 5, NCCL_SUM = 0, NCCL_MAX = 2, NCCL_MIN = 3;

// dlopen libnccl once; RAPID_ENCCL if it or a required symbol is missing
int32_t load_nccl();

struct Comm {
    int device = 0, rank = 0, world = 1;
    nccl_comm comm = nullptr;
};

#define RAPID_NCCL(call)                                                                                              \
    do {                                                                                                              \
        int _r = (call);                                                                                              \
        if (_r != 0) { set_error("NCCL error %d (%s): %s", _r, g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?", #call); return RAPID_ENCCL; } \
    } while (0)

}  // namespace rapid

struct rapid_comm : rapid::Comm {};
