// TMA (cp.async.bulk.tensor) staging of image tiles into shared memory, sm_90a.
//
// Every u8 image buffer a tile kernel reads has a row pitch that is a multiple of 16 bytes (plf_pitch16), which makes
// any halo tile of any image of a batch a legal box of a 3-D tensor map {x: width, y: height, z: image} with strides
// {1, pitch, image stride}.  One elected thread issues ONE bulk-tensor copy per CTA (SASS: UTMALDG.3D) that lands the
// (tile + halo) box in shared memory and signals an mbarrier with the byte count; the other threads only wait on the
// barrier - no per-thread address arithmetic, no funnel shifts, no st.shared.  Every box STARTS on a 16-byte boundary of
// global memory (the kernels use no other x origin; y and z are free because the strides are multiples of 16), so the
// tile grids are shifted: a kernel whose tile needs columns from
// x0 - R places its tiles at x0 = 64 * bx - (16 - R) (plf_tma_x0), or loads a wider box from the aligned address below
// its origin and indexes it with the remainder (FAST).  Elements of the box that lie outside the
// image come back as zeros; kernels that need BORDER_REFLECT_101 patch those cells from the in-image part of the same
// tile (plf_tma_reflect_fix: shared memory -> shared memory, border CTAs only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

static inline int plf_pitch16(int w) { return (w + 15) & ~15; }
// number of 64-column tiles when the tile grid is shifted left by (16 - R) columns (see above)
static inline int plf_tma_tiles_x(int w, int R) { return (w + (16 - R) + 63) / 64; }

// Host: tensor map over nimg images of w x h bytes, row pitch `pitch`, image stride `img_stride` (both multiples of
// 16), box = box_w x box_h x 1 (box_w a multiple of 16).  The driver entry point is resolved through the runtime so
// that the library keeps linking against the static CUDA runtime only.
static inline bool plf_tma_encode_u8(CUtensorMap* map, const void* base, int w, int h, int nimg, size_t pitch,
                                     size_t img_stride, int box_w, int box_h) {
  typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static encode_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return false;
    fn = (encode_fn)p;
  }
  if ((pitch & 15) || (img_stride & 15) || (box_w & 15) || ((uintptr_t)base & 15) || box_w > 256 || box_h > 256) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)nimg};
  const cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)img_stride};
  const cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Host: the tensor maps of one kernel over caller-owned images, two entries keyed by source pointer and geometry (the
// batched pipeline alternates between two upload buffers).  An entry is reused while its image count covers the
// request; otherwise the least recently used entry is re-encoded.  The box is the owner's and fixed for its lifetime.
struct PlfTmaCache {
  struct Entry {
    const void* src = nullptr;
    int w = 0, h = 0, nimg = 0;
    size_t pitch = 0, img_stride = 0;
    CUtensorMap map;
  };
  Entry e[2];
  int last = 1;   // entry used by the previous call
  // The map over images [0, nimg) of src, or nullptr if encoding fails.
  const CUtensorMap* get(const void* src, int w, int h, int nimg, size_t pitch, size_t img_stride, int box_w, int box_h) {
    for (int k = 0; k < 2; ++k) {
      const Entry& c = e[k];
      if (c.src == src && c.w == w && c.h == h && c.pitch == pitch && c.img_stride == img_stride && c.nimg >= nimg) {
        last = k;
        return &c.map;
      }
    }
    last ^= 1;
    Entry& c = e[last];
    c = Entry();
    if (!plf_tma_encode_u8(&c.map, src, w, h, nimg, pitch, img_stride, box_w, box_h)) return nullptr;
    c.src = src; c.w = w; c.h = h; c.nimg = nimg; c.pitch = pitch; c.img_stride = img_stride;
    return &c.map;
  }
};

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t plf_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One thread: initialise the barrier for one arrival and make the initialisation visible to the async proxy.
__device__ __forceinline__ void plf_mbar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(plf_smem_u32(bar)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// One thread: expect `bytes`, then issue the 3-D box load (x, y, z may be negative / run past the image: zero fill).
__device__ __forceinline__ void plf_tma_load_3d(void* smem_dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar,
                                                uint32_t bytes) {
  const uint32_t b = plf_smem_u32(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          plf_smem_u32(smem_dst)),
      "l"(map), "r"(x), "r"(y), "r"(z), "r"(b)
      : "memory");
}
// All threads: wait for phase `parity` of the barrier.
__device__ __forceinline__ void plf_mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t b = plf_smem_u32(bar);
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(b),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ int plf_reflect101(int i, int n) {
  if (n == 1) return 0;
  while (i < 0 || i >= n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
  }
  return i;
}
// BORDER_REFLECT_101 for a TMA-staged tile: raw[ry][rx] holds pixel (gx0 + rx, gy0 + ry), zeros outside the w x h image.
// Cells outside the image are rewritten from their mirror pixel, which lies inside this same tile (the caller's halo
// is smaller than its tile; asserted by the callers' geometry); columns first on in-image rows, then whole rows.
// Call by all threads of the CTA between the barrier wait and the first use; contains the __syncthreads it needs.
template <int RH, int RP>
__device__ __forceinline__ void plf_tma_reflect_fix(uint8_t (*raw)[RP], int gx0, int gy0, int w, int h, int need_w) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int ry_lo = max(0, -gy0), ry_hi = min(RH, h - gy0);   // in-image rows of the tile: [ry_lo, ry_hi)
  const bool colfix = gx0 < 0 || gx0 + need_w > w;
  if (colfix) {
    for (int i = tid; i < (ry_hi - ry_lo) * need_w; i += nt) {
      const int ry = ry_lo + i / need_w, rx = i - (i / need_w) * need_w;
      const int gx = gx0 + rx;
      if (gx < 0 || gx >= w) {
        const int m = plf_reflect101(gx, w) - gx0;     // mirror column; outside the tile only for cells no output uses
        if (m >= 0 && m < RP) raw[ry][rx] = raw[ry][m];
      }
    }
    __syncthreads();
  }
  if (ry_lo > 0 || ry_hi < RH) {
    const int nrows = ry_lo + (RH - ry_hi);
    for (int i = tid; i < nrows * need_w; i += nt) {
      const int k = i / need_w, rx = i - k * need_w;
      const int ry = k < ry_lo ? k : ry_hi + (k - ry_lo);
      const int m = plf_reflect101(gy0 + ry, h) - gy0;
      if (m >= 0 && m < RH) raw[ry][rx] = raw[m][rx];
    }
  }
}
#endif
