// shard_comm.cpp -- see shard_comm.h
#include "shard_comm.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include "cuda_owned.h"
#include <nccl.h>   // types and enums only: every function is resolved with dlsym

#include <cstring>
#include <mutex>

namespace lama_b200 {

namespace {
struct Nccl {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    std::string err;
};

Nccl* nccl(std::string& err)
{
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        // a libnccl already in the process (e.g. the one torch brought) is reused; otherwise the system library is loaded
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            n.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (n.lib) break;
        }
        if (!n.lib) { n.err = std::string("cannot load libnccl.so.2: ") + dlerror(); return; }
        auto sym = [&](const char* s) -> void* {
            void* p = dlsym(n.lib, s);
            if (!p && n.err.empty()) n.err = std::string("libnccl lacks ") + s;
            return p;
        };
        n.GetUniqueId    = reinterpret_cast<decltype(n.GetUniqueId)>(sym("ncclGetUniqueId"));
        n.CommInitRank   = reinterpret_cast<decltype(n.CommInitRank)>(sym("ncclCommInitRank"));
        n.CommDestroy    = reinterpret_cast<decltype(n.CommDestroy)>(sym("ncclCommDestroy"));
        n.AllGather      = reinterpret_cast<decltype(n.AllGather)>(sym("ncclAllGather"));
        n.Send           = reinterpret_cast<decltype(n.Send)>(sym("ncclSend"));
        n.Recv           = reinterpret_cast<decltype(n.Recv)>(sym("ncclRecv"));
        n.GroupStart     = reinterpret_cast<decltype(n.GroupStart)>(sym("ncclGroupStart"));
        n.GroupEnd       = reinterpret_cast<decltype(n.GroupEnd)>(sym("ncclGroupEnd"));
        n.GetErrorString = reinterpret_cast<decltype(n.GetErrorString)>(sym("ncclGetErrorString"));
    });
    if (!n.err.empty()) { err = n.err; return nullptr; }
    return &n;
}
}  // namespace

struct ShardComm {
    Nccl* n = nullptr;
    ncclComm_t comm = nullptr;
    lama_b200::Stream stream;
    int rank = 0, world = 1, device = 0;
    uint64_t collectives = 0;
    std::string err;
    int fail(const std::string& what, ncclResult_t r) { err = what + ": " + (n && n->GetErrorString ? n->GetErrorString(r) : "nccl error"); return -2; }
    int cfail(const std::string& what, cudaError_t e) { err = what + ": " + cudaGetErrorString(e); return -2; }
};

int shard_unique_id(uint8_t id[128], std::string& err)
{
    Nccl* n = nccl(err);
    if (!n) return -2;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId");
    ncclUniqueId u;
    ncclResult_t r = n->GetUniqueId(&u);
    if (r != ncclSuccess) { err = std::string("ncclGetUniqueId: ") + n->GetErrorString(r); return -2; }
    std::memcpy(id, &u, 128);
    return 0;
}

ShardComm* shard_comm_create(const uint8_t id[128], int rank, int world, int device, std::string& err)
{
    Nccl* n = nccl(err);
    if (!n) return nullptr;
    if (cudaSetDevice(device) != cudaSuccess) { err = "shard_comm_create: bad device"; return nullptr; }
    ShardComm* c = new ShardComm();
    c->n = n; c->rank = rank; c->world = world; c->device = device;
    ncclUniqueId u;
    std::memcpy(&u, id, 128);
    ncclResult_t r = n->CommInitRank(&c->comm, world, u, rank);
    if (r != ncclSuccess) { err = std::string("ncclCommInitRank: ") + n->GetErrorString(r); delete c; return nullptr; }
    // its own stream: the engine's stream holds the running map update, which the exchange of the match results must not wait for
    if (c->stream.create() != cudaSuccess) { err = "shard_comm_create: no stream"; n->CommDestroy(c->comm); delete c; return nullptr; }
    return c;
}

void shard_comm_destroy(ShardComm* c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    c->stream.reset();
    if (c->comm) c->n->CommDestroy(c->comm);
    delete c;
}
void* shard_stream(ShardComm* c) { return c->stream.get(); }
int shard_world(const ShardComm* c) { return c->world; }
int shard_rank(const ShardComm* c) { return c->rank; }
const std::string& shard_error(const ShardComm* c) { return c->err; }
uint64_t shard_collectives(const ShardComm* c) { return c->collectives; }

int shard_allgather(ShardComm* c, const void* d_send, void* d_recv, size_t bytes)
{
    ncclResult_t r = c->n->AllGather(d_send, d_recv, bytes, ncclChar, c->comm, c->stream);
    if (r != ncclSuccess) return c->fail("ncclAllGather", r);
    ++c->collectives;
    return 0;
}

int shard_exchange(ShardComm* c, const std::vector<ShardXfer>& sends, const std::vector<ShardXfer>& recvs)
{
    if (sends.empty() && recvs.empty()) return 0;
    ncclResult_t r = c->n->GroupStart();
    if (r != ncclSuccess) return c->fail("ncclGroupStart", r);
    for (const ShardXfer& x : sends) {
        r = c->n->Send(x.dptr, x.bytes, ncclChar, x.peer, c->comm, c->stream);
        if (r != ncclSuccess) return c->fail("ncclSend", r);
    }
    for (const ShardXfer& x : recvs) {
        r = c->n->Recv(x.dptr, x.bytes, ncclChar, x.peer, c->comm, c->stream);
        if (r != ncclSuccess) return c->fail("ncclRecv", r);
    }
    r = c->n->GroupEnd();
    if (r != ncclSuccess) return c->fail("ncclGroupEnd", r);
    ++c->collectives;
    return 0;
}

int shard_sync(ShardComm* c)
{
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return c->cfail("cudaStreamSynchronize(comm)", e);
    return 0;
}

}  // namespace lama_b200
