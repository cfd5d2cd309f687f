// libptk runtime: error state, driver-API binding, NVRTC JIT, module/launch, CUDA graphs, events, memcpy.
// Host-side only; the kernels live in the other translation units and in the JIT templates.
#include <dlfcn.h>
#include <nvrtc.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <string>
#include <vector>
#include "ptk_common.h"

namespace ptk {

static thread_local std::string g_err;
static DriverApi g_drv;
static bool g_init = false;
static int g_device = -1;
static int g_sms = 0;
static std::mutex g_mu;

void set_error(const std::string& msg) { g_err = msg; }
ptk_status fail(ptk_status code, const std::string& msg) {
  g_err = msg;
  return code;
}
ptk_status check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return PTK_OK;
  g_err = std::string(what) + ": " + cudaGetErrorName(e) + ": " + cudaGetErrorString(e);
  cudaGetLastError();  // clear the sticky-less error so the next call starts clean
  return PTK_ERR_CUDA;
}
ptk_status check_cu(CUresult r, const char* what) {
  if (r == CUDA_SUCCESS) return PTK_OK;
  const char* s = nullptr;
  if (g_drv.GetErrorString) g_drv.GetErrorString(r, &s);
  g_err = std::string(what) + ": CUresult " + std::to_string((int)r) + (s ? std::string(": ") + s : "");
  return PTK_ERR_CUDA;
}
const DriverApi& drv() { return g_drv; }
bool initialised() { return g_init; }
int sm_count() { return g_sms; }

template <typename F>
static ptk_status bind(F& slot, const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || p == nullptr || q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return fail(PTK_ERR_CUDA, std::string("cannot bind driver entry point ") + name);
  }
  slot = reinterpret_cast<F>(p);
  return PTK_OK;
}

// ---- NVRTC, bound lazily with dlopen so that libptk.so loads on a box without the toolkit libraries ------------
struct Nvrtc {
  void* h = nullptr;
  nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*);
  nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*);
  nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*);
  nvrtcResult (*GetProgramLog)(nvrtcProgram, char*);
  nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*);
  nvrtcResult (*GetCUBIN)(nvrtcProgram, char*);
  nvrtcResult (*DestroyProgram)(nvrtcProgram*);
  const char* (*GetErrorString)(nvrtcResult);
};
static Nvrtc g_rtc;

static ptk_status load_nvrtc() {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_rtc.h) return PTK_OK;
  const char* cands[] = {"/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so.12", "libnvrtc.so", nullptr};
  void* h = nullptr;
  for (int i = 0; cands[i] && !h; ++i) h = dlopen(cands[i], RTLD_NOW | RTLD_LOCAL);
  if (!h) return fail(PTK_ERR_NVRTC, std::string("cannot dlopen libnvrtc: ") + dlerror());
#define PTK_SYM(field, name)                                                                   \
  *(void**)(&g_rtc.field) = dlsym(h, name);                                                   \
  if (!g_rtc.field) return fail(PTK_ERR_NVRTC, std::string("libnvrtc lacks symbol ") + name);
  PTK_SYM(CreateProgram, "nvrtcCreateProgram")
  PTK_SYM(CompileProgram, "nvrtcCompileProgram")
  PTK_SYM(GetProgramLogSize, "nvrtcGetProgramLogSize")
  PTK_SYM(GetProgramLog, "nvrtcGetProgramLog")
  PTK_SYM(GetCUBINSize, "nvrtcGetCUBINSize")
  PTK_SYM(GetCUBIN, "nvrtcGetCUBIN")
  PTK_SYM(DestroyProgram, "nvrtcDestroyProgram")
  PTK_SYM(GetErrorString, "nvrtcGetErrorString")
#undef PTK_SYM
  g_rtc.h = h;
  return PTK_OK;
}

}  // namespace ptk

using namespace ptk;

extern "C" {

int ptk_version(void) { return 100; }
const char* ptk_last_error(void) { return g_err.c_str(); }

ptk_status ptk_init(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_init && device == g_device) return PTK_OK;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(PTK_ERR_CUDA, "ptk_init: no CUDA device visible (libptk has no CPU fallback)");
  }
  if (device < 0 || device >= n) return fail(PTK_ERR_ARG, "ptk_init: bad device ordinal");
  PTK_CUDA(cudaSetDevice(device));
  PTK_CUDA(cudaFree(0));
  cudaDeviceProp prop;
  PTK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    return fail(PTK_ERR_UNSUPPORTED, std::string("ptk_init: device '") + prop.name +
                                         "' is not sm_90 class; libptk is built for sm_90a (H100) only");
  }
  g_sms = prop.multiProcessorCount;
  ptk_status s;
  if ((s = bind(g_drv.GetErrorString, "cuGetErrorString")) != PTK_OK) return s;
  if ((s = bind(g_drv.ModuleLoadDataEx, "cuModuleLoadDataEx")) != PTK_OK) return s;
  if ((s = bind(g_drv.ModuleUnload, "cuModuleUnload")) != PTK_OK) return s;
  if ((s = bind(g_drv.ModuleGetFunction, "cuModuleGetFunction")) != PTK_OK) return s;
  if ((s = bind(g_drv.LaunchKernelEx, "cuLaunchKernelEx")) != PTK_OK) return s;
  if ((s = bind(g_drv.FuncSetAttribute, "cuFuncSetAttribute")) != PTK_OK) return s;
  if ((s = bind(g_drv.OccupancyMaxActiveBlocksPerMultiprocessor,
                "cuOccupancyMaxActiveBlocksPerMultiprocessor")) != PTK_OK) return s;
  if ((s = bind(g_drv.TensorMapEncodeTiled, "cuTensorMapEncodeTiled")) != PTK_OK) return s;
  g_device = device;
  g_init = true;
  return PTK_OK;
}

int ptk_sm_count(void) { return g_sms; }
int ptk_device(void) { return g_device; }

ptk_status ptk_sync_stream(void* stream) {
  PTK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_memcpy_h2d_async(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes == 0) return PTK_OK;
  PTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_memcpy_d2h_async(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes == 0) return PTK_OK;
  PTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_memcpy_d2d_async(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes == 0) return PTK_OK;
  PTK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_memset_async(void* dst, int byte, size_t bytes, void* stream) {
  if (bytes == 0) return PTK_OK;
  PTK_CUDA(cudaMemsetAsync(dst, byte, bytes, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_host_alloc_pinned(void** out, size_t bytes) {
  PTK_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return PTK_OK;
}
ptk_status ptk_host_free_pinned(void* p) {
  PTK_CUDA(cudaFreeHost(p));
  return PTK_OK;
}

// ---- JIT -----------------------------------------------------------------------------------------------------------
void ptk_free(void* p) { free(p); }

ptk_status ptk_jit_compile(const char* src, const char* const* opts, int n_opts, void** cubin, size_t* cubin_size,
                           char** log) {
  if (log) *log = nullptr;
  if (!src || !cubin || !cubin_size) return fail(PTK_ERR_ARG, "ptk_jit_compile: null argument");
  ptk_status s = load_nvrtc();
  if (s != PTK_OK) return s;
  nvrtcProgram prog;
  nvrtcResult r = g_rtc.CreateProgram(&prog, src, "ptk_jit.cu", 0, nullptr, nullptr);
  if (r != NVRTC_SUCCESS) return fail(PTK_ERR_NVRTC, std::string("nvrtcCreateProgram: ") + g_rtc.GetErrorString(r));
  std::vector<const char*> o;
  o.push_back("--gpu-architecture=sm_90a");
  o.push_back("--std=c++17");
  o.push_back("-lineinfo");
  o.push_back("-default-device");
  for (int i = 0; i < n_opts; ++i) o.push_back(opts[i]);
  r = g_rtc.CompileProgram(prog, (int)o.size(), o.data());
  size_t lsz = 0;
  g_rtc.GetProgramLogSize(prog, &lsz);
  std::string lg;
  if (lsz > 1) {
    lg.resize(lsz);
    g_rtc.GetProgramLog(prog, &lg[0]);
    if (log) *log = strdup(lg.c_str());
  }
  if (r != NVRTC_SUCCESS) {
    g_rtc.DestroyProgram(&prog);
    return fail(PTK_ERR_NVRTC, std::string("nvrtcCompileProgram: ") + g_rtc.GetErrorString(r) + "\n" + lg);
  }
  size_t sz = 0;
  g_rtc.GetCUBINSize(prog, &sz);
  char* img = (char*)malloc(sz ? sz : 1);
  g_rtc.GetCUBIN(prog, img);
  g_rtc.DestroyProgram(&prog);
  *cubin = img;
  *cubin_size = sz;
  return PTK_OK;
}

ptk_status ptk_module_load(const void* image, size_t size, void** module) {
  PTK_REQUIRE_INIT();
  (void)size;
  CUmodule m;
  PTK_CU(g_drv.ModuleLoadDataEx(&m, image, 0, nullptr, nullptr));
  *module = (void*)m;
  return PTK_OK;
}
ptk_status ptk_module_unload(void* module) {
  PTK_REQUIRE_INIT();
  PTK_CU(g_drv.ModuleUnload((CUmodule)module));
  return PTK_OK;
}
ptk_status ptk_module_get_function(void* module, const char* name, void** func) {
  PTK_REQUIRE_INIT();
  CUfunction f;
  PTK_CU(g_drv.ModuleGetFunction(&f, (CUmodule)module, name));
  *func = (void*)f;
  return PTK_OK;
}
ptk_status ptk_func_set_max_dynamic_smem(void* func, int bytes) {
  PTK_REQUIRE_INIT();
  PTK_CU(g_drv.FuncSetAttribute((CUfunction)func, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, bytes));
  return PTK_OK;
}
ptk_status ptk_func_max_active_blocks(void* func, int block_threads, int dyn_smem, int* out) {
  PTK_REQUIRE_INIT();
  PTK_CU(g_drv.OccupancyMaxActiveBlocksPerMultiprocessor(out, (CUfunction)func, block_threads, (size_t)dyn_smem));
  return PTK_OK;
}

ptk_status ptk_launch(void* func, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by, unsigned bz,
                      unsigned dyn_smem, void* stream, void** args, int flags, int cluster_x) {
  PTK_REQUIRE_INIT();
  if (gx == 0 || gy == 0 || gz == 0) return PTK_OK;  // empty launch = nothing to do (zero-size tensors)
  CUlaunchConfig cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDimX = gx; cfg.gridDimY = gy; cfg.gridDimZ = gz;
  cfg.blockDimX = bx; cfg.blockDimY = by; cfg.blockDimZ = bz;
  cfg.sharedMemBytes = dyn_smem;
  cfg.hStream = (CUstream)stream;
  CUlaunchAttribute attrs[2];
  unsigned na = 0;
  if (flags & 1) {
    attrs[na].id = CU_LAUNCH_ATTRIBUTE_COOPERATIVE;
    attrs[na].value.cooperative = 1;
    ++na;
  }
  if (cluster_x > 1) {
    attrs[na].id = CU_LAUNCH_ATTRIBUTE_CLUSTER_DIMENSION;
    attrs[na].value.clusterDim.x = (unsigned)cluster_x;
    attrs[na].value.clusterDim.y = 1;
    attrs[na].value.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = na;
  PTK_CU(g_drv.LaunchKernelEx(&cfg, (CUfunction)func, args, nullptr));
  return PTK_OK;
}

// ---- graphs ----------------------------------------------------------------------------------------------------------
ptk_status ptk_graph_begin_capture(void* stream) {
  PTK_CUDA(cudaStreamBeginCapture((cudaStream_t)stream, cudaStreamCaptureModeRelaxed));
  return PTK_OK;
}
ptk_status ptk_graph_end_capture(void* stream, void** graph_exec) {
  cudaGraph_t g = nullptr;
  PTK_CUDA(cudaStreamEndCapture((cudaStream_t)stream, &g));
  cudaGraphExec_t ge = nullptr;
  cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  PTK_CUDA(e);
  *graph_exec = (void*)ge;
  return PTK_OK;
}
ptk_status ptk_graph_launch(void* graph_exec, void* stream) {
  PTK_CUDA(cudaGraphLaunch((cudaGraphExec_t)graph_exec, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_graph_destroy(void* graph_exec) {
  PTK_CUDA(cudaGraphExecDestroy((cudaGraphExec_t)graph_exec));
  return PTK_OK;
}

// ---- events ----------------------------------------------------------------------------------------------------------
ptk_status ptk_event_create(void** ev) {
  cudaEvent_t e;
  PTK_CUDA(cudaEventCreate(&e));
  *ev = (void*)e;
  return PTK_OK;
}
ptk_status ptk_event_record(void* ev, void* stream) {
  PTK_CUDA(cudaEventRecord((cudaEvent_t)ev, (cudaStream_t)stream));
  return PTK_OK;
}
ptk_status ptk_event_elapsed_ms(void* start, void* stop, float* ms) {
  PTK_CUDA(cudaEventSynchronize((cudaEvent_t)stop));
  PTK_CUDA(cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop));
  return PTK_OK;
}
ptk_status ptk_event_destroy(void* ev) {
  PTK_CUDA(cudaEventDestroy((cudaEvent_t)ev));
  return PTK_OK;
}
ptk_status ptk_stream_wait_event(void* stream, void* ev) {
  PTK_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)ev, 0));
  return PTK_OK;
}

}  // extern "C"
