// Data-movement kernels of the IMPALA ResNet trunk (polybeast_learner.py:134-266), templated on the
// activation element type T (float for the fp32 backend, __nv_bfloat16 for the tensor-core backend).
// All activations are NHWC; every kernel moves 16-byte vectors (VEC = 16/sizeof(T) channels).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace tb {

template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void unpack(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
template <> struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& v, float* f) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 t = __bfloat1622float2(h[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint4 o;
    __nv_bfloat162 p0 = __floats2bfloat162_rn(f[0], f[1]), p1 = __floats2bfloat162_rn(f[2], f[3]);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(f[4], f[5]), p3 = __floats2bfloat162_rn(f[6], f[7]);
    o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
    o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
    return o;
  }
};

// x [N,H,W,C] -> col [N*H*W, ldk], k = (kh*3 + kw)*C + c, 3x3 window, stride 1, zero padding 1.
// relu_in: the conv consumes relu(x) (residual blocks: nn.ReLU() precedes each conv, pl:165-183).
template <typename T>
int im2col3x3(const T* x, T* col, int64_t N, int H, int W, int C, int64_t ldk, int relu_in, cudaStream_t stream);

// first conv of the net: frames u8 NCHW [N,C,H,W] -> patch matrix, k = (c*3 + kh)*3 + kw (the reference
// weight's own flattening).  TOut = uint8_t (fp32 backend: x/255 applied on read) or bf16 (exact 0..255).
template <typename TOut>
int im2col3x3_u8_nchw(const uint8_t* frame, TOut* col, int64_t N, int C, int H, int W, int64_t ldk, cudaStream_t stream);

// dcol [N*H*W, ldk] -> dx [N,H,W,C] (gather form): dx = gather(dcol) * (relu_src > 0 if relu_src) + addend
template <typename T>
int col2im3x3(const T* dcol, const T* relu_src, const T* addend, T* dx, int64_t N, int H, int W, int C, int64_t ldk,
              cudaStream_t stream);

// nn.MaxPool2d(kernel_size=3, stride=2, padding=1) forward / backward (first-maximum tie rule)
// forward also records the argmax tap (0..8) of every output element; backward gathers through it
template <typename T>
int maxpool3x3s2_fwd(const T* x, T* y, uint8_t* argmax, int64_t N, int H, int W, int C, cudaStream_t stream);
template <typename T>
int maxpool3x3s2_bwd(const uint8_t* argmax, const T* dy, T* dx, int64_t N, int H, int W, int C, cudaStream_t stream);

// y = relu(x) (elementwise, n elements); dx = dy * (x > 0) + (addend ? addend : 0)
template <typename T>
int relu_fwd(const T* x, T* y, int64_t n, cudaStream_t stream);
template <typename T>
int relu_bwd(const T* x, const T* dy, T* dx, int64_t n, cudaStream_t stream);

// column sums of a T matrix (bias gradients) - fp32 accumulation
template <typename T>
int colsum_t(const T* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream);

// fp32 [rows, cols] (ld) -> T [rows, ldo] (zero padded); T == float is a strided copy
template <typename T>
int convert_from_f32(const float* in, T* out, int64_t rows, int64_t cols, int64_t ld, int64_t ldo, cudaStream_t stream);

}  // namespace tb
