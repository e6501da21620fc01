// Thin shim over the CUDA driver API and NVRTC.  Both libraries are dlopen'ed on first
// use so libgandiva_b200.so loads (and Make() can still generate + compile kernels with
// NVRTC) on a box without a GPU driver; anything that needs a device fails loudly with
// GDV_CUDA_ERROR.  No CUDA runtime (cudart) dependency: the host side talks to the
// driver directly (BASELINE.json north_star: "Host is C++ calling the CUDA driver").
#pragma once
#include <cuda.h>
#include <nvrtc.h>

#include <string>
#include <vector>

#include "gdv_codegen.h"

namespace gdv {

struct DriverApi {
  bool loaded = false;
  std::string load_error;
  CUresult (*Init)(unsigned int);
  CUresult (*DeviceGetCount)(int*);
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  CUresult (*DevicePrimaryCtxRetain)(CUcontext*, CUdevice);
  CUresult (*CtxSetCurrent)(CUcontext);
  CUresult (*CtxGetCurrent)(CUcontext*);
  CUresult (*MemAlloc)(CUdeviceptr*, size_t);
  CUresult (*MemFree)(CUdeviceptr);
  CUresult (*MemHostAlloc)(void**, size_t, unsigned int);
  CUresult (*MemFreeHost)(void*);
  CUresult (*MemcpyHtoDAsync)(CUdeviceptr, const void*, size_t, CUstream);
  CUresult (*MemcpyDtoHAsync)(void*, CUdeviceptr, size_t, CUstream);
  CUresult (*MemcpyDtoDAsync)(CUdeviceptr, CUdeviceptr, size_t, CUstream);
  CUresult (*MemsetD8Async)(CUdeviceptr, unsigned char, size_t, CUstream);
  CUresult (*StreamCreate)(CUstream*, unsigned int);
  CUresult (*StreamSynchronize)(CUstream);
  CUresult (*StreamDestroy)(CUstream);
  CUresult (*StreamWaitEvent)(CUstream, CUevent, unsigned int);
  CUresult (*EventCreate)(CUevent*, unsigned int);
  CUresult (*EventRecord)(CUevent, CUstream);
  CUresult (*EventSynchronize)(CUevent);
  CUresult (*EventDestroy)(CUevent);
  CUresult (*ModuleLoadData)(CUmodule*, const void*);
  CUresult (*ModuleUnload)(CUmodule);
  CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*);
  CUresult (*FuncGetAttribute)(int*, CUfunction_attribute, CUfunction);
  CUresult (*FuncSetAttribute)(CUfunction, CUfunction_attribute, int);
  CUresult (*OccupancyMaxActiveBlocksPerMultiprocessor)(int*, CUfunction, int, size_t);
  CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned,
                           unsigned, CUstream, void**, void**);
  CUresult (*GetErrorString)(CUresult, const char**);
  CUresult (*PointerGetAttribute)(void*, CUpointer_attribute, CUdeviceptr);
  CUresult (*CtxEnablePeerAccess)(CUcontext, unsigned int);
  CUresult (*DeviceCanAccessPeer)(int*, CUdevice, CUdevice);
  CUresult (*IpcGetMemHandle)(CUipcMemHandle*, CUdeviceptr);
  CUresult (*IpcOpenMemHandle)(CUdeviceptr*, CUipcMemHandle, unsigned int);
  CUresult (*IpcCloseMemHandle)(CUdeviceptr);
  CUresult (*MemGetAddressRange)(CUdeviceptr*, size_t*, CUdeviceptr);
};
// Loads libcuda.so.1 and calls cuInit(0) once.  Returns nullptr-safe struct; check .loaded.
const DriverApi& Driver();
Status CuCheck(CUresult r, const char* what);

struct NvrtcApi {
  bool loaded = false;
  std::string load_error;
  nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*,
                               const char* const*);
  nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*);
  nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*);
  nvrtcResult (*GetProgramLog)(nvrtcProgram, char*);
  nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*);
  nvrtcResult (*GetCUBIN)(nvrtcProgram, char*);
  nvrtcResult (*GetPTXSize)(nvrtcProgram, size_t*);
  nvrtcResult (*GetPTX)(nvrtcProgram, char*);
  nvrtcResult (*DestroyProgram)(nvrtcProgram*);
  const char* (*GetErrorString)(nvrtcResult);
};
const NvrtcApi& Nvrtc();

// The device function library text (gdv_device_lib.cuh), embedded at build time.
extern "C" const char gdv_device_lib_text[];
extern "C" const unsigned long long gdv_device_lib_text_len;
// Precompiled (nvcc, sm_90a) cubin of device/static_kernels.cu, embedded at build time.
extern "C" const unsigned char gdv_static_kernels_cubin[];
extern "C" const unsigned long long gdv_static_kernels_cubin_len;

// Compile `source` (which #includes "gdv_device_lib.cuh") to an sm_90a cubin.
Status CompileToCubin(const std::string& source, const std::string& arch, bool optimize,
                      bool want_ptx, std::vector<char>* cubin, std::string* ptx,
                      std::string* log);

}  // namespace gdv
