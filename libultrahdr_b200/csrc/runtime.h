// Device runtime: per-device LUT residency, a grow-only arena per worker (device + pinned host)
// and a stream.  180 GB of HBM per GPU means we never free inside a codec call: arenas are
// rewound, not released.
#pragma once
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <mutex>
#include <string>
#include <vector>

namespace uhdr_b200 {

// uhdr_codec_err_t values
enum : int { E_OK = 0, E_ERROR = 1, E_UNKNOWN = 2, E_INVALID_PARAM = 3, E_MEM = 4,
             E_INVALID_OP = 5, E_UNSUPPORTED = 6 };

void set_last_error(const std::string& s);
const char* last_error();
int fail(int code, const char* fmt, ...);

#define CUDA_TRY(expr)                                                                     \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return ::uhdr_b200::fail(_e == cudaErrorMemoryAllocation ? E_MEM : E_ERROR,          \
                               "CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e),      \
                               __FILE__, __LINE__, #expr);                                 \
  } while (0)

// Copy that has landed when it returns, for tables uploaded once and then read by kernels on any stream.  A plain
// cudaMemcpy from pageable memory (or device to device) may return before its DMA completes, and it is ordered
// only against the legacy stream: kernels on the library's non-blocking streams could read the table before it.
int copy_sync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind);

// ---- per-device kernel state ---------------------------------------------------------------------
// Constant tables in device memory and wave sizes are made once per device, on its first use, and kept for the life
// of the process.  A slot is constant-initialised: a function-local `static PerDevice<T>` has no init guard and makes
// no heap call.  Looking a value up costs one cudaGetDevice and one acquire load; only the first use on a device
// takes the slot's lock.  A device ordinal >= kMaxDevices is an error.
constexpr int kMaxDevices = 64;
template <class T>
struct PerDevice {
  std::atomic<T> v[kMaxDevices] = {};  // T{}: not made yet on that device (the initialiser keeps the slot constexpr)
  std::mutex mu;
};

// CTAs of one full wave of `kernel` on the current device: SMs x co-resident CTAs per SM (1 when the occupancy query
// fails).  A kernel launched with more than 48 KiB of dynamic shared memory is opted in to `dyn_smem` on each device
// first.  Returns 0 + sets last error on failure.
int wave_ctas(PerDevice<int>& slot, const void* kernel, int threads, size_t dyn_smem);
// A constant table of `bytes` on the current device: build(host) fills it on the host, copy_sync uploads it.  With
// `symbol` (a __device__ / __constant__ variable) the table is copied there; otherwise it gets its own allocation.
// Returns the device address, or nullptr + sets last error.
const void* device_table(PerDevice<const void*>& slot, size_t bytes, void (*build)(void* host),
                         const void* symbol = nullptr);
// out[0] = device tables made, out[1] = wave sizes asked of the runtime, since process start
void device_state_stats(unsigned long long out[2]);

// Device-resident LUT blob for the current device (built on first use, or installed from a
// broadcast).  Returns nullptr + sets last error when no CUDA device is usable.
const float* device_luts();
int install_luts_from_device(const void* dptr);
int read_back_luts(float* host_out);

void set_kernel_timing(bool on);
bool kernel_timing_enabled();
// "name count total_ms\n" lines; resets the accumulators when `reset`
std::string kernel_timing_report(bool reset);

#define TIMED(ws, name, call)        \
  do {                               \
    (ws).t_begin(name);              \
    cudaError_t _te = (call);        \
    (ws).t_end();                    \
    CUDA_TRY(_te);                   \
  } while (0)

struct PhaseTrace {  // UHDR_B200_TRACE=1: wall-clock phases of one call on stderr
  bool on = getenv("UHDR_B200_TRACE") != nullptr;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  void mark(const char* what) {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    fprintf(stderr, "[uhdr_b200] %-26s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  }
};

// release every parked arena block back to the driver; returns the bytes freed
size_t trim_parked_blocks();

class Arena {
 public:
  // min_block: the smallest block taken from the driver (0: 64 MiB of device / 32 MiB of pinned memory)
  explicit Arena(bool pinned_host, size_t min_block = 0) : pinned_(pinned_host), min_block_(min_block) {}
  ~Arena();
  void* alloc(size_t bytes, size_t align = 256);  // nullptr on failure (last error set)
  void rewind();
  // keep everything allocated so far, release what comes later (inputs stay resident while the
  // per-encode scratch is recycled)
  void set_floor();
  void clear_floor();
  size_t reserved() const;

 private:
  struct Block { char* base; size_t size, used, floor; };
  std::vector<Block> blocks_;
  bool pinned_;
  size_t min_block_;
  int device_ = -1;  // device the blocks belong to (set at the first allocation)
};

class Workspace {
 public:
  Workspace();
  ~Workspace();
  int init();  // binds to the current device, creates the stream
  cudaStream_t stream() const { return ext_stream_set_ ? ext_stream_ : stream_; }
  // run the following calls on a caller-owned stream (the *_dev stage entry points); clear_external_stream()
  // returns to the workspace's own
  void use_external_stream(cudaStream_t s) { ext_stream_ = s; ext_stream_set_ = true; }
  void clear_external_stream() { ext_stream_set_ = false; }
  void* dalloc(size_t bytes) { return dev_.alloc(bytes); }
  void* halloc(size_t bytes) { return host_.alloc(bytes); }
  void rewind() { dev_.rewind(); host_.rewind(); }
  void set_floor() { dev_.set_floor(); host_.set_floor(); }
  void clear_floor() { dev_.clear_floor(); host_.clear_floor(); }
  // per-kernel CUDA-event timing (enabled globally with set_kernel_timing); begin/end bracket one
  // launch on this workspace's stream, collect() must run after the stream was synchronised
  void t_begin(const char* name);
  void t_end();
  void t_collect();
  const float* luts() const { return luts_; }
  int sync();

 private:
  Arena dev_{false}, host_{true};
  cudaStream_t stream_ = nullptr;
  cudaStream_t ext_stream_ = nullptr;
  cudaEvent_t sync_ev_ = nullptr;   // UHDR_B200_BLOCKING_SYNC=1: sync() sleeps on this event instead of spinning
  bool ext_stream_set_ = false;
  const float* luts_ = nullptr;
  int device_ = -1;
  struct Span { const char* name; cudaEvent_t a, b; };
  std::vector<Span> spans_;
  std::vector<cudaEvent_t> ev_pool_;
  cudaEvent_t get_event();
};

}  // namespace uhdr_b200
