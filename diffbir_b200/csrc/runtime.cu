// Host-side runtime of libdiffbir_b200.so: error plumbing, device info, TMA descriptor
// encoding through the driver entry point (no link-time dependency on libcuda).
#include "common.cuh"
#include "../../include/diffbir_b200.h"
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <string.h>
#include <stdlib.h>

static thread_local char g_err[1024] = "";

void dbir_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* dbir_last_error(void) { return g_err; }
extern "C" const char* dbir_version(void) {
  return "diffbir_b200 0.1 (sm_90a; wgmma/TMA)";
}
extern "C" int dbir_operand_kind(void) { return DBIR_OPERAND_KIND; }
extern "C" int dbir_pdl_enabled(void) {
  static const int on = [] { const char* e = getenv("DBIR_PDL"); return e ? atoi(e) : 1; }();
  return on;
}

extern "C" int dbir_sm_count(void) {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int dbir_make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes,
                   int swizzle128) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    dbir_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return -1;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    dbir_set_error("TMA base pointer %p is not 16-byte aligned", base);
    return -1;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i - 1];
      if (gstr[i - 1] % 16 != 0) {
        dbir_set_error("TMA stride %llu (dim %d) is not a multiple of 16 bytes",
                       (unsigned long long)gstr[i - 1], i);
        return -1;
      }
    }
  }
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                         : elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_UINT32
                                           : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUresult r = enc(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr,
                   bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 == 1 ? CU_TENSOR_MAP_SWIZZLE_128B
                   : swizzle128 == 2 ? CU_TENSOR_MAP_SWIZZLE_64B
                   : swizzle128 == 3 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    dbir_set_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d, dims %llu/%llu, box %u/%u)",
                   (int)r, rank, (unsigned long long)dims[0],
                   (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
    return -1;
  }
  return 0;
}
