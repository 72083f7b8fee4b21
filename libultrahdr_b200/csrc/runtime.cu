#include "runtime.h"

#include <cstdarg>
#include <cstdlib>
#include <atomic>
#include <cstdio>
#include <new>
#include <map>
#include <mutex>

#include "tables.h"

namespace uhdr_b200 {

static thread_local std::string g_err;
void set_last_error(const std::string& s) { g_err = s; }
const char* last_error() { return g_err.c_str(); }
int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

int copy_sync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
  cudaStream_t s = nullptr;
  CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  cudaError_t e = cudaMemcpyAsync(dst, src, bytes, kind, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaStreamDestroy(s);
  CUDA_TRY(e);
  return E_OK;
}

// ---- per-device kernel state --------------------------------------------------------------------
namespace {
std::atomic<unsigned long long> g_state_made[2];  // device tables, wave sizes

// the slot's value for the current device; make(dev, &value) runs once per device, under the slot's lock (kernels
// are launched from many host threads at once)
template <class T, class Make>
int per_device(PerDevice<T>& slot, T* out, Make make) {
  int dev = -1;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) return fail(E_ERROR, "device ordinal %d out of range", dev);
  T v = slot.v[dev].load(std::memory_order_acquire);
  if (!v) {
    std::lock_guard<std::mutex> lk(slot.mu);
    v = slot.v[dev].load(std::memory_order_relaxed);
    if (!v) {
      if (int rc = make(dev, &v)) return rc;
      slot.v[dev].store(v, std::memory_order_release);
    }
  }
  *out = v;
  return E_OK;
}
}  // namespace

int wave_ctas(PerDevice<int>& slot, const void* kernel, int threads, size_t dyn_smem) {
  int ctas = 0;
  const int err = per_device(slot, &ctas, [&](int dev, int* out) -> int {
    // function attributes belong to the device's context: every device needs its own opt-in
    if (dyn_smem > (48 << 10))
      CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem));
    int sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, dyn_smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    *out = per_sm * (sms > 0 ? sms : 132);
    g_state_made[1].fetch_add(1, std::memory_order_relaxed);
    return E_OK;
  });
  return err ? 0 : ctas;
}

const void* device_table(PerDevice<const void*>& slot, size_t bytes, void (*build)(void* host), const void* symbol) {
  const void* table = nullptr;
  const int err = per_device(slot, &table, [&](int, const void** out) -> int {
    std::vector<unsigned char> host(bytes);
    build(host.data());
    void* d = nullptr;
    if (symbol) CUDA_TRY(cudaGetSymbolAddress(&d, symbol));
    else CUDA_TRY(cudaMalloc(&d, bytes));
    if (int rc = copy_sync(d, host.data(), bytes, cudaMemcpyHostToDevice)) {
      if (!symbol) cudaFree(d);
      return rc;
    }
    *out = d;
    g_state_made[0].fetch_add(1, std::memory_order_relaxed);
    return E_OK;
  });
  return err ? nullptr : table;
}

void device_state_stats(unsigned long long out[2]) {
  for (int i = 0; i < 2; i++) out[i] = g_state_made[i].load(std::memory_order_relaxed);
}

// ---- LUT residency ------------------------------------------------------------------------------
static std::mutex g_lut_mu;
static std::map<int, float*> g_luts;  // device ordinal -> device blob

static float* lut_slot(int dev) {
  auto it = g_luts.find(dev);
  if (it != g_luts.end()) return it->second;
  float* d = nullptr;
  if (cudaMalloc(&d, sizeof(float) * kLutTotalFloats) != cudaSuccess) return nullptr;
  g_luts[dev] = d;
  return d;
}

const float* device_luts() {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    fail(E_ERROR, "no usable CUDA device: %s (libuhdr_b200 has no CPU fallback)", cudaGetErrorString(e));
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(g_lut_mu);
  auto it = g_luts.find(dev);
  if (it != g_luts.end()) return it->second;
  float* d = lut_slot(dev);
  if (!d) {
    fail(E_MEM, "cudaMalloc of LUT blob failed");
    return nullptr;
  }
  std::vector<float> host(kLutTotalFloats);
  build_lut_blob(host.data());
  if (copy_sync(d, host.data(), sizeof(float) * kLutTotalFloats, cudaMemcpyHostToDevice) != E_OK) return nullptr;
  return d;
}

int install_luts_from_device(const void* dptr) {
  int dev = -1;
  CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_lut_mu);
  float* d = lut_slot(dev);
  if (!d) return fail(E_MEM, "cudaMalloc of LUT blob failed");
  // on the legacy stream, after the broadcast that filled dptr; landed before any kernel of ours reads it
  CUDA_TRY(cudaMemcpy(d, dptr, sizeof(float) * kLutTotalFloats, cudaMemcpyDeviceToDevice));
  CUDA_TRY(cudaStreamSynchronize(cudaStreamLegacy));
  return E_OK;
}

int read_back_luts(float* host_out) {
  const float* d = device_luts();
  if (!d) return E_ERROR;
  CUDA_TRY(cudaMemcpy(host_out, d, sizeof(float) * kLutTotalFloats, cudaMemcpyDeviceToHost));
  return E_OK;
}

// ---- arenas -------------------------------------------------------------------------------------
// Blocks of released arenas are parked in a process-wide cache instead of going back to the driver:
// the reference's usage pattern is create handle / run / release per image, and pinning a few
// hundred MB of host memory (or cudaMalloc of as much HBM) costs far more than the decode itself.
namespace {
struct ParkedBlock { char* base; size_t size; int device; };
std::mutex g_park_mu;
std::vector<ParkedBlock> g_parked[2];              // [0] device memory, [1] pinned host memory
size_t g_parked_bytes[2] = {0, 0};
constexpr size_t kParkCap[2] = {(size_t)8 << 30, (size_t)4 << 30};

char* take_parked(bool pinned, int device, size_t bytes, size_t max_size, size_t* got) {
  std::lock_guard<std::mutex> lk(g_park_mu);
  auto& v = g_parked[pinned ? 1 : 0];
  int best = -1;
  for (int i = 0; i < (int)v.size(); i++) {
    if (v[i].size < bytes || (!pinned && v[i].device != device)) continue;
    if (best < 0 || v[i].size < v[best].size) best = i;
  }
  // a handle of the same kind asks for the same block sizes in the same order, so near-exact matches
  // are the rule; handing a much larger block to a small request would only force the next large
  // request back to the driver
  if (best < 0 || v[best].size > max_size) return nullptr;
  char* base = v[best].base;
  *got = v[best].size;
  g_parked_bytes[pinned ? 1 : 0] -= v[best].size;
  v.erase(v.begin() + best);
  return base;
}
bool park(bool pinned, int device, char* base, size_t size) {
  std::lock_guard<std::mutex> lk(g_park_mu);
  const int k = pinned ? 1 : 0;
  if (g_parked_bytes[k] + size > kParkCap[k]) return false;
  g_parked[k].push_back({base, size, device});
  g_parked_bytes[k] += size;
  return true;
}
}  // namespace

size_t trim_parked_blocks() {
  std::vector<ParkedBlock> take[2];
  {
    std::lock_guard<std::mutex> lk(g_park_mu);
    for (int k = 0; k < 2; k++) {
      take[k].swap(g_parked[k]);
      g_parked_bytes[k] = 0;
    }
  }
  size_t freed = 0;
  int cur = -1;
  cudaGetDevice(&cur);
  for (auto& b : take[0]) {
    if (b.device >= 0 && b.device != cur) cudaSetDevice(b.device);
    cudaFree(b.base);
    freed += b.size;
    if (b.device >= 0 && b.device != cur && cur >= 0) cudaSetDevice(cur);
  }
  for (auto& b : take[1]) {
    cudaFreeHost(b.base);
    freed += b.size;
  }
  return freed;
}

// Callers (Workspace) drain their stream before the arenas go away: a parked block may be handed to
// another handle on another stream at once, and unlike cudaFree parking does not synchronise.
Arena::~Arena() {
  for (auto& b : blocks_) {
    if (park(pinned_, device_, b.base, b.size)) continue;
    if (pinned_) cudaFreeHost(b.base);
    else cudaFree(b.base);
  }
}
void* Arena::alloc(size_t bytes, size_t align) {
  if (bytes == 0) bytes = 1;
  for (auto& b : blocks_) {
    size_t off = (b.used + align - 1) / align * align;
    if (off + bytes <= b.size) {
      b.used = off + bytes;
      return b.base + off;
    }
  }
  const size_t min_block = min_block_ ? min_block_ : pinned_ ? (size_t)32 << 20 : (size_t)64 << 20;
  size_t sz = bytes > min_block ? bytes : min_block;
  sz = (sz + 4095) / 4096 * 4096;
  if (device_ < 0) cudaGetDevice(&device_);
  // an exactly sized arena (min_block set: a resident image, kept for long) takes a parked block only if it is
  // nearly the size asked for
  const size_t max_size = min_block_ ? sz + sz / 32 : sz + sz / 4 + ((size_t)1 << 20);
  char* base = take_parked(pinned_, device_, sz, max_size, &sz);
  if (!base) {
    cudaError_t e = pinned_ ? cudaHostAlloc((void**)&base, sz, cudaHostAllocPortable)
                            : cudaMalloc((void**)&base, sz);
    if (e != cudaSuccess) {
      fail(E_MEM, "%s of %zu bytes failed: %s", pinned_ ? "cudaHostAlloc" : "cudaMalloc", sz,
           cudaGetErrorString(e));
      return nullptr;
    }
  }
  blocks_.push_back({base, sz, bytes, 0});
  return base;
}
void Arena::rewind() {
  for (auto& b : blocks_) b.used = b.floor;
}
void Arena::set_floor() {
  for (auto& b : blocks_) b.floor = b.used;
}
void Arena::clear_floor() {
  for (auto& b : blocks_) b.floor = b.used = 0;
}
size_t Arena::reserved() const {
  size_t s = 0;
  for (auto& b : blocks_) s += b.size;
  return s;
}

Workspace::Workspace() {}
Workspace::~Workspace() {
  if (stream_) {
    // error returns can leave kernels / async copies in flight on this stream; they must have
    // finished before the arena blocks (destroyed after this body) are parked for other handles
    cudaStreamSynchronize(stream_);
    cudaStreamDestroy(stream_);
  }
  for (auto& s : spans_) { cudaEventDestroy(s.a); cudaEventDestroy(s.b); }
  for (cudaEvent_t e : ev_pool_) cudaEventDestroy(e);
  if (sync_ev_) cudaEventDestroy(sync_ev_);
}
int Workspace::init() {
  if (stream_) return E_OK;
  luts_ = device_luts();
  if (!luts_) return E_ERROR;
  CUDA_TRY(cudaGetDevice(&device_));
  CUDA_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  return E_OK;
}
// A host thread waiting for its stream normally spins (lowest latency).  With many handles per GPU and several GPUs
// per host that is one busy core per waiting thread; UHDR_B200_BLOCKING_SYNC=1 makes the wait a sleep on an event
// created with cudaEventBlockingSync (a few tens of microseconds more per wait, no core burnt).
static bool blocking_sync_wanted() {
  static const bool on = [] { const char* e = getenv("UHDR_B200_BLOCKING_SYNC"); return e && *e && *e != '0'; }();
  return on;
}
int Workspace::sync() {
  if (blocking_sync_wanted()) {
    if (!sync_ev_) CUDA_TRY(cudaEventCreateWithFlags(&sync_ev_, cudaEventBlockingSync | cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(sync_ev_, stream()));
    CUDA_TRY(cudaEventSynchronize(sync_ev_));
  } else {
    CUDA_TRY(cudaStreamSynchronize(stream()));
  }
  if (!spans_.empty()) t_collect();
  return E_OK;
}
// ---- kernel timing ------------------------------------------------------------------------------
static std::atomic<bool> g_timing{false};
static std::mutex g_timing_mu;
struct TimingAcc { unsigned long long n = 0; double total = 0, mn = 1e30, mx = 0; };
static std::map<std::string, TimingAcc> g_timing_acc;
void set_kernel_timing(bool on) { g_timing = on; }
bool kernel_timing_enabled() { return g_timing; }
std::string kernel_timing_report(bool reset) {
  std::lock_guard<std::mutex> lk(g_timing_mu);
  std::string out;
  char line[256];
  for (auto& kv : g_timing_acc) {
    snprintf(line, sizeof line, "%s %llu %.6f %.6f %.6f\n", kv.first.c_str(), kv.second.n, kv.second.total, kv.second.mn, kv.second.mx);
    out += line;
  }
  if (reset) g_timing_acc.clear();
  return out;
}
cudaEvent_t Workspace::get_event() {
  if (!ev_pool_.empty()) {
    cudaEvent_t e = ev_pool_.back();
    ev_pool_.pop_back();
    return e;
  }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
void Workspace::t_begin(const char* name) {
  if (!g_timing) return;
  Span s{name, get_event(), get_event()};
  cudaEventRecord(s.a, stream());
  spans_.push_back(s);
}
void Workspace::t_end() {
  if (!g_timing || spans_.empty()) return;
  cudaEventRecord(spans_.back().b, stream());
}
void Workspace::t_collect() {
  std::lock_guard<std::mutex> lk(g_timing_mu);
  for (auto& s : spans_) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, s.a, s.b) == cudaSuccess) {
      auto& acc = g_timing_acc[s.name];
      acc.n++;
      acc.total += ms;
      if (ms < acc.mn) acc.mn = ms;
      if (ms > acc.mx) acc.mx = ms;
    }
    ev_pool_.push_back(s.a);
    ev_pool_.push_back(s.b);
  }
  spans_.clear();
}

}  // namespace uhdr_b200
