// gs_nccl.h -- NCCL bound at run time (dlopen), so libgsplat_b200.so has no link-time dependency on it: single-GPU hosts
// load the library on machines without NCCL, and inside a process that already carries a libnccl (PyTorch bundles one)
// the group path uses THAT copy instead of loading a second one.
//
// Only the handful of entry points the group path needs are declared, with the prototypes of nccl.h (2.x ABI).
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stddef.h>

namespace gs {

typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef enum { ncclSuccess = 0 } ncclResult_t;
typedef enum { ncclInt8 = 0, ncclChar = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3 } ncclDataType_t;

struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int *) = nullptr;
  bool ok() const { return lib != nullptr; }
};

inline const NcclApi &nccl_api() {
  static NcclApi api = [] {
    NcclApi a;
    // a copy that is already mapped (e.g. torch's) wins; else the system one
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return a;
#define GS_NCCL_SYM(field, name) *(void **)(&a.field) = dlsym(h, name)
    GS_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
    GS_NCCL_SYM(CommInitRank, "ncclCommInitRank");
    GS_NCCL_SYM(CommInitAll, "ncclCommInitAll");
    GS_NCCL_SYM(CommDestroy, "ncclCommDestroy");
    GS_NCCL_SYM(AllGather, "ncclAllGather");
    GS_NCCL_SYM(Broadcast, "ncclBroadcast");
    GS_NCCL_SYM(GroupStart, "ncclGroupStart");
    GS_NCCL_SYM(GroupEnd, "ncclGroupEnd");
    GS_NCCL_SYM(GetErrorString, "ncclGetErrorString");
    GS_NCCL_SYM(GetVersion, "ncclGetVersion");
#undef GS_NCCL_SYM
    if (a.GetUniqueId && a.CommInitRank && a.CommInitAll && a.CommDestroy && a.AllGather && a.Broadcast &&
        a.GroupStart && a.GroupEnd && a.GetErrorString)
      a.lib = h;
    return a;
  }();
  return api;
}

}  // namespace gs
