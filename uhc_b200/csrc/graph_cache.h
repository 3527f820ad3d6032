// graph_cache.h -- the cache of captured CUDA graphs shared by the rollout (rollout.cu), the evaluation (eval.cu) and the tracker
// (track.cu).  Host only, not part of the C ABI.
//
// A graph holds the kernel parameters of its capture by value.  Its key is every argument that reaches a kernel, as an opaque byte
// string the caller builds by appending PODs (zeroed first: the padding is compared too).  Pointers the caller does not pass but the
// graph still holds (the engine view, scratch buffers) are covered by generation counters stored with the entry: drop_stale destroys
// every graph captured under other generations, since it can never be replayed again.  At `cap` entries the oldest one is evicted.
#pragma once
#include <cuda_runtime.h>
#include <array>
#include <string>
#include <utility>
#include <vector>
#include "errors.h"

namespace uhc {

class GraphCache {
public:
    using Gens = std::array<unsigned long long, 3>;
    explicit GraphCache(size_t cap) : cap_(cap) {}
    template <class T> static void append(std::string *key, const T *p, size_t count = 1) { key->append((const char *)p, count * sizeof(T)); }

    void clear() { for (Entry &g : entries_) cudaGraphExecDestroy(g.exec); entries_.clear(); }
    void drop_stale(const Gens &gens) {
        for (size_t i = 0; i < entries_.size();) {
            if (entries_[i].gens != gens) { cudaGraphExecDestroy(entries_[i].exec); entries_.erase(entries_.begin() + i); } else i++;
        }
    }
    cudaGraphExec_t find(const std::string &key) const {
        for (const Entry &g : entries_) if (g.key == key) return g.exec;
        return nullptr;
    }
    // enqueue(stream) -> 0 or its error code, run under capture on a private stream (a legacy-stream capture is not allowed; the replay
    // is ordered by the stream it is launched on).  Returns enqueue's code unchanged, with the error text it left, or -1 with the CUDA
    // error in uhc_err().
    template <class Enqueue> static int capture(Enqueue &&enqueue, cudaGraphExec_t *exec) {
        cudaStream_t cs; cudaGraph_t graph = nullptr;
        cudaError_t ce = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
        if (ce != cudaSuccess) { uhc_err() = std::string("cudaStreamCreateWithFlags: ") + cudaGetErrorString(ce); return -1; }
        int rc = 0; const char *what = "begin of the stream capture";
        ce = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
        if (ce == cudaSuccess) {
            rc = enqueue(cs);
            what = "cudaStreamEndCapture"; ce = cudaStreamEndCapture(cs, &graph);
        }
        cudaStreamDestroy(cs);
        if (rc == 0 && ce == cudaSuccess) { what = "cudaGraphInstantiate"; ce = cudaGraphInstantiate(exec, graph, 0); }
        if (graph) cudaGraphDestroy(graph);
        if (rc) return rc;
        if (ce != cudaSuccess) { uhc_err() = std::string(what) + ": " + cudaGetErrorString(ce); return -1; }
        return 0;
    }
    void insert(std::string key, const Gens &gens, cudaGraphExec_t exec) {
        if (entries_.size() >= cap_) { cudaGraphExecDestroy(entries_.front().exec); entries_.erase(entries_.begin()); }
        entries_.push_back(Entry{std::move(key), gens, exec});
    }

private:
    struct Entry { std::string key; Gens gens; cudaGraphExec_t exec; };
    size_t cap_;
    std::vector<Entry> entries_;
};

}  // namespace uhc
