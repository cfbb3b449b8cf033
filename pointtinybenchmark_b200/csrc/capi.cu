// Library-level entry points of libptb_b200.so (error string, ABI version, launch counter) and the per-stream scratch blocks.
#include "ptb_common.cuh"
#include <map>
#include <mutex>
#include <utility>

namespace ptb {
thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

static std::mutex g_scratch_mu;
static std::map<std::pair<int, void*>, StreamScratch*> g_scratch;

StreamScratch* stream_scratch(void* stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    fail("%s", "stream_scratch: cudaGetDevice failed");
    return nullptr;
  }
  std::lock_guard<std::mutex> lock(g_scratch_mu);
  auto key = std::make_pair(dev, stream);
  auto it = g_scratch.find(key);
  if (it != g_scratch.end()) return it->second;
  StreamScratch* p = nullptr;
  // zeroed on the stream that owns the block: a plain cudaMemset of device memory is queued on the legacy default stream, which a
  // non-blocking stream's first kernel does not wait for
  if (cudaMalloc(&p, sizeof(StreamScratch)) != cudaSuccess ||
      cudaMemsetAsync(p, 0, sizeof(StreamScratch), (cudaStream_t)stream) != cudaSuccess) {
    cudaGetLastError();
    fail("%s", "stream_scratch: cudaMalloc / cudaMemset of the per-stream scratch block failed");
    return nullptr;
  }
  g_scratch[key] = p;
  return p;
}
}  // namespace ptb

extern "C" int ptb_abi_version(void) { return PTB_ABI_VERSION; }
extern "C" const char* ptb_last_error(void) { return ptb::g_err; }
extern "C" uint64_t ptb_launch_count(void) { return ptb::g_launches.load(); }

extern "C" int ptb_reset_stream_state(void* stream) {
  ptb::StreamScratch* p = ptb::stream_scratch(stream);
  if (!p) return 1;
  if (cudaMemsetAsync(p, 0, sizeof(ptb::StreamScratch), (cudaStream_t)stream) != cudaSuccess)
    return ptb::fail("%s", "ptb_reset_stream_state: cudaMemsetAsync failed");
  return 0;
}
