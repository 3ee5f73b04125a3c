// SPDX-License-Identifier: Apache-2.0
// Host-side helpers shared by the translation units of libhcpb200: thread-local error string,
// and CUtensorMap construction through the driver entry point (no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

namespace hcp {

int set_error(int code, const char* msg);
int set_cuda_error(cudaError_t e, const char* where);
// streaming multiprocessors of the current device (queried once); launch planning sizes its waves by it
int num_sms();

// bf16, SWIZZLE_128B, zero fill for out-of-bounds elements.  `dims`/`box` innermost first;
// `strides_bytes` has rank-1 entries (the innermost stride is the element size).
int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, bool swizzle128 = true);

// [rows, inner] row-major matrix with row pitch `ld` elements; box = box_inner x box_rows.
inline int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t ld,
                        uint32_t box_inner, uint32_t box_rows) {
    uint64_t dims[2] = {inner, rows};
    uint64_t strides[1] = {ld * 2};
    uint32_t box[2] = {box_inner, box_rows};
    return make_tmap_nd(out, base, 2, dims, strides, box);
}

// Geometry of the 3x3 / pad 1 convolutions on NHWC bf16 activations (forward, dgrad and both weight-gradient kernels).
// One 128-row M tile is a box of bw x bh pixels x bn images of the tile grid (tH x tW pixels per image): whole 128-pixel row pieces,
// whole rows, or whole images.  The grid of such boxes is tiles_w x tiles_h per image (bn == 1) or ceil(B / bn) tiles (bn > 1).
struct ConvBox {
    int32_t bw, bh, bn, tiles_w, tiles_h;
};
// Plans the box of a tH x tW tile grid; on failure the error message starts with `who`.
int plan_conv_box(int64_t tH, int64_t tW, const char* who, ConvBox& box);
// TMA map of x [B, H, W, C] whose boxes are 64 channels x one ConvBox: 4-D for stride 1, for stride 2 the 5-D phase view
// [B][H/2][2][W/2][2C] (input row 2*oh + kh - 1 and column 2*ow + kw - 1 become (phase, index) pairs of the view).
int make_tmap_nhwc(CUtensorMap* out, const void* x, int64_t B, int64_t H, int64_t W, int64_t C, int stride, const ConvBox& box);
// Shift of tap (kh, kw) in the map above: added to the channel, W, H coordinates of the box and, 5-D only, the H phase.
struct ConvTap {
    int32_t c0_off, dw, dh, c2;
};
ConvTap conv_tap(int kh, int kw, int stride, int64_t C);

// true when every pointer is 16-byte aligned (NULL counts as aligned): the elementwise kernels load and store uint4 / float4
template <typename... P>
inline bool aligned16(const P*... p) {
    return ((((uintptr_t)p) | ... | (uintptr_t)0) & 15) == 0;
}

// Launch with programmatic stream serialization (PDL): the kernel may start while its predecessor on the stream drains; every
// kernel of the library calls pdl_wait() (common.cuh) before touching global memory.  HCP_PDL=0 turns the attribute off.
bool pdl_enabled();
void note_launch();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    note_launch();
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Launch as thread-block clusters of `cluster_x` CTAs along x (gridDim.x must be a multiple of it).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, unsigned cluster_x,
                                  Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster_x;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    note_launch();
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace hcp
