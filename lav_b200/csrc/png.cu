// Batched decode of the recordings' 8-bit grayscale PNG maps (BasicDataset.load_bev's cv2.imdecode(..., IMREAD_GRAYSCALE),
// lav/utils/datasets/basic_dataset.py:94,99) on the device: one warp per image, several images per CTA.  The host has walked the
// chunks (signature, IHDR, CRCs) and packed each image's concatenated IDAT payload, i.e. its zlib stream, into one buffer;
// png_inflate.cuh inflates it straight into the destination plane and undoes the row filters there.
#include <algorithm>

#include "common.cuh"
#include "png_inflate.cuh"

namespace {

struct PngJob {             // 32 bytes, layout documented in lav_b200.h
  long long off, len;       // the zlib stream: bytes [off, off + len) of the source buffer
  int dst, h, w, pad;       // destination plane; the image size from IHDR
};
static_assert(sizeof(PngJob) == 32, "PngJob layout is part of the ABI (lav_b200.h)");

constexpr int kWarps = 4;

__host__ __device__ constexpr int warp_smem(int h) { return (int)((sizeof(lavb_png::Scratch) + h + 15) / 16 * 16); }

__global__ void __launch_bounds__(kWarps * 32) png_decode_gray8_kernel(const uint8_t* __restrict__ src, long long src_bytes,
                                                                       const PngJob* __restrict__ jobs, int n_jobs,
                                                                       uint8_t* __restrict__ out, int n_planes, int h, int w,
                                                                       int* __restrict__ status) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int warp = threadIdx.x >> 5;
  uint8_t* mine = smem + warp * warp_smem(h);
  lavb_png::Scratch& s = *reinterpret_cast<lavb_png::Scratch*>(mine);
  uint8_t* filt = mine + sizeof(lavb_png::Scratch);
  const lavb_png::Lanes L{(int)(threadIdx.x & 31), 32};
  for (int j = blockIdx.x * kWarps + warp; j < n_jobs; j += gridDim.x * kWarps) {
    const PngJob job = jobs[j];
    int st;
    if (job.off < 0 || job.len < 0 || job.off > src_bytes || job.len > src_bytes - job.off || job.dst < 0 || job.dst >= n_planes ||
        job.h != h || job.w != w) {
      st = lavb_png::kBadJob;
    } else {
      st = lavb_png::decode_gray8(s, filt, src + job.off, job.len, out + (size_t)job.dst * h * w, h, w, L);
    }
    if (L.lane == 0) status[j] = st;
    __syncwarp();
  }
}

}  // namespace

extern "C" int lavb_png_decode_gray8(const uint8_t* d_src, long long src_bytes, const void* d_jobs, int n_jobs, uint8_t* d_out,
                                     int n_planes, int h, int w, int* d_status, void* stream) {
  LAVB_CHECK_ARG(n_jobs >= 0 && n_planes >= 0 && src_bytes >= 0 && h > 0 && w > 0 && h <= 4096 && w <= 4096,
                 "png_decode_gray8: bad arguments");
  if (n_jobs == 0) return 0;
  const int smem = kWarps * warp_smem(h);
  LAVB_CUDA_OK(lavb::ensure_dyn_smem((const void*)png_decode_gray8_kernel, smem));
  const int grid = (int)std::min<long long>(lavb::ceil_div(n_jobs, kWarps), 64LL * kNumSMs);
  png_decode_gray8_kernel<<<grid, kWarps * 32, smem, (cudaStream_t)stream>>>(
      d_src, src_bytes, reinterpret_cast<const PngJob*>(d_jobs), n_jobs, d_out, n_planes, h, w, d_status);
  LAVB_LAUNCH_OK();
  return 0;
}
