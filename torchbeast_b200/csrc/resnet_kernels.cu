// See resnet_kernels.cuh.  HBM-bound gathers on 16-byte vectors; grid-stride loops; no tensor cores.
#include "resnet_kernels.cuh"

#include "gemm_tc.cuh"
#include "net_kernels.cuh"

namespace tb {

static inline unsigned rgrid(int64_t work, int threads) {
  int64_t blocks = (work + threads - 1) / threads;
  const int64_t cap = int64_t(kNumSMs) * 16;
  if (blocks > cap) blocks = cap;
  return (unsigned)(blocks < 1 ? 1 : blocks);
}

template <typename T>
__global__ void im2col3x3_kernel(const uint4* __restrict__ x, uint4* __restrict__ col, int64_t N, int H, int W, int CV,
                                 int64_t ldkv, int relu_in) {
  // one thread = one 16-byte vector of one (pixel, tap)
  const int64_t total = N * H * W * 9 * CV;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int cv = int(i % CV);
    int64_t t = i / CV;
    const int tap = int(t % 9); t /= 9;
    const int ox = int(t % W); t /= W;
    const int oy = int(t % H);
    const int64_t n = t / H;
    const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      v = __ldg(x + ((n * H + iy) * W + ix) * CV + cv);
      if (relu_in) {
        float f[Vec16<T>::N];
        Vec16<T>::unpack(v, f);
#pragma unroll
        for (int j = 0; j < Vec16<T>::N; ++j) f[j] = fmaxf(f[j], 0.0f);
        v = Vec16<T>::pack(f);
      }
    }
    col[((n * H + oy) * W + ox) * ldkv + int64_t(tap) * CV + cv] = v;
  }
}

template <typename T>
int im2col3x3(const T* x, T* col, int64_t N, int H, int W, int C, int64_t ldk, int relu_in, cudaStream_t stream) {
  ProfScope prof("im2col3x3", stream);
  constexpr int V = Vec16<T>::N;
  TB_REQUIRE(C % V == 0 && ldk % V == 0, "im2col3x3: C and ldk must be multiples of %d", V);
  const int64_t total = N * H * W * 9 * (C / V);
  if (total == 0) return 0;
  im2col3x3_kernel<T><<<rgrid(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(col), N,
                                                              H, W, C / V, ldk / V, relu_in);
  return check_launch("im2col3x3_kernel");
}
template int im2col3x3<float>(const float*, float*, int64_t, int, int, int, int64_t, int, cudaStream_t);
template int im2col3x3<__nv_bfloat16>(const __nv_bfloat16*, __nv_bfloat16*, int64_t, int, int, int, int64_t, int, cudaStream_t);

template <typename TOut> __device__ __forceinline__ TOut from_u8(uint8_t v);
template <> __device__ __forceinline__ uint8_t from_u8<uint8_t>(uint8_t v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_u8<__nv_bfloat16>(uint8_t v) { return __float2bfloat16_rn(float(v)); }

template <typename TOut>
__global__ void im2col3x3_u8_nchw_kernel(const uint8_t* __restrict__ frame, TOut* __restrict__ col, int64_t N, int C, int H,
                                         int W, int64_t ldk) {
  // one thread = one output pixel: gathers its C x 3 x 3 neighbourhood (neighbouring threads share cache
  // lines) and writes its whole patch row with wide stores
  const int64_t total = N * H * W;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int ox = int(i % W);
    int64_t t = i / W;
    const int oy = int(t % H);
    const int64_t n = t / H;
    uint8_t v[40];
#pragma unroll
    for (int k = 0; k < 40; ++k) v[k] = 0;
    for (int c = 0; c < C && c < 4; ++c) {
      const uint8_t* src = frame + (n * C + c) * H * W;
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v[c * 9 + tap] = __ldg(src + iy * W + ix);
      }
    }
    TOut* dst = col + i * ldk;
    if constexpr (sizeof(TOut) == 2) {
      if (ldk == 40) {
        uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          uint4 o;
          uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            __nv_bfloat162 p = __floats2bfloat162_rn(float(v[q * 8 + 2 * e]), float(v[q * 8 + 2 * e + 1]));
            ow[e] = *reinterpret_cast<uint32_t*>(&p);
          }
          d4[q] = o;
        }
        continue;
      }
    }
    for (int k = 0; k < C * 9; ++k) dst[k] = from_u8<TOut>(v[k]);
  }
}

template <typename TOut>
int im2col3x3_u8_nchw(const uint8_t* frame, TOut* col, int64_t N, int C, int H, int W, int64_t ldk, cudaStream_t stream) {
  ProfScope prof("im2col3x3_u8", stream);
  TB_REQUIRE(C <= 4, "im2col3x3_u8_nchw: at most 4 input channels");
  const int64_t total = N * H * W;
  if (total == 0) return 0;
  if (ldk > int64_t(C) * 9 && !(sizeof(TOut) == 2 && ldk == 40)) {  // zero the k padding (the vector path writes it itself)
    cudaError_t e = cudaMemsetAsync(col, 0, size_t(N) * H * W * ldk * sizeof(TOut), stream);
    TB_REQUIRE(e == cudaSuccess, "im2col3x3_u8: memset: %s", cudaGetErrorString(e));
  }
  im2col3x3_u8_nchw_kernel<TOut><<<rgrid(total, 128), 128, 0, stream>>>(frame, col, N, C, H, W, ldk);
  return check_launch("im2col3x3_u8_nchw_kernel");
}
template int im2col3x3_u8_nchw<uint8_t>(const uint8_t*, uint8_t*, int64_t, int, int, int, int64_t, cudaStream_t);
template int im2col3x3_u8_nchw<__nv_bfloat16>(const uint8_t*, __nv_bfloat16*, int64_t, int, int, int, int64_t, cudaStream_t);

template <typename T>
__global__ void col2im3x3_kernel(const uint4* __restrict__ dcol, const uint4* __restrict__ relu_src,
                                 const uint4* __restrict__ addend, uint4* __restrict__ dx, int64_t N, int H, int W, int CV,
                                 int64_t ldkv) {
  constexpr int V = Vec16<T>::N;
  const int64_t total = N * H * W * CV;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int cv = int(i % CV);
    int64_t t = i / CV;
    const int ix = int(t % W); t /= W;
    const int iy = int(t % H);
    const int64_t n = t / H;
    float s[V];
#pragma unroll
    for (int j = 0; j < V; ++j) s[j] = 0.0f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      // output pixel (oy, ox) reads input (oy + kh - 1, ox + kw - 1): oy = iy - kh + 1
      const int oy = iy - tap / 3 + 1, ox = ix - tap % 3 + 1;
      if (oy < 0 || oy >= H || ox < 0 || ox >= W) continue;
      float f[V];
      Vec16<T>::unpack(__ldg(dcol + ((n * H + oy) * W + ox) * ldkv + int64_t(tap) * CV + cv), f);
#pragma unroll
      for (int j = 0; j < V; ++j) s[j] += f[j];
    }
    if (relu_src) {
      float f[V];
      Vec16<T>::unpack(__ldg(relu_src + i), f);
#pragma unroll
      for (int j = 0; j < V; ++j) s[j] = f[j] > 0.0f ? s[j] : 0.0f;
    }
    if (addend) {
      float f[V];
      Vec16<T>::unpack(__ldg(addend + i), f);
#pragma unroll
      for (int j = 0; j < V; ++j) s[j] += f[j];
    }
    dx[i] = Vec16<T>::pack(s);
  }
}

template <typename T>
int col2im3x3(const T* dcol, const T* relu_src, const T* addend, T* dx, int64_t N, int H, int W, int C, int64_t ldk,
              cudaStream_t stream) {
  ProfScope prof("col2im3x3", stream);
  constexpr int V = Vec16<T>::N;
  TB_REQUIRE(C % V == 0 && ldk % V == 0, "col2im3x3: C and ldk must be multiples of %d", V);
  const int64_t total = N * H * W * (C / V);
  if (total == 0) return 0;
  col2im3x3_kernel<T><<<rgrid(total, 256), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(dcol), reinterpret_cast<const uint4*>(relu_src), reinterpret_cast<const uint4*>(addend),
      reinterpret_cast<uint4*>(dx), N, H, W, C / V, ldk / V);
  return check_launch("col2im3x3_kernel");
}
template int col2im3x3<float>(const float*, const float*, const float*, float*, int64_t, int, int, int, int64_t, cudaStream_t);
template int col2im3x3<__nv_bfloat16>(const __nv_bfloat16*, const __nv_bfloat16*, const __nv_bfloat16*, __nv_bfloat16*, int64_t,
                                      int, int, int, int64_t, cudaStream_t);

template <typename T>
__global__ void maxpool_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, uint8_t* __restrict__ arg, int64_t N,
                                   int H, int W, int OH, int OW, int CV) {
  // also records, per output element, which of the 9 window taps held the FIRST maximum (torch's rule)
  constexpr int V = Vec16<T>::N;
  const int64_t total = N * OH * OW * CV;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int cv = int(i % CV);
    int64_t t = i / CV;
    const int ox = int(t % OW); t /= OW;
    const int oy = int(t % OH);
    const int64_t n = t / OH;
    float m[V];
    uint8_t a[V];
#pragma unroll
    for (int j = 0; j < V; ++j) { m[j] = -INFINITY; a[j] = 0; }
    for (int kh = 0; kh < 3; ++kh) {
      const int iy = oy * 2 + kh - 1;
      if (iy < 0 || iy >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int ix = ox * 2 + kw - 1;
        if (ix < 0 || ix >= W) continue;
        float f[V];
        Vec16<T>::unpack(__ldg(x + ((n * H + iy) * W + ix) * CV + cv), f);
#pragma unroll
        for (int j = 0; j < V; ++j)
          if (f[j] > m[j]) { m[j] = f[j]; a[j] = uint8_t(kh * 3 + kw); }
      }
    }
    y[i] = Vec16<T>::pack(m);
#pragma unroll
    for (int j = 0; j < V; ++j) arg[i * V + j] = a[j];
  }
}

template <typename T>
__global__ void maxpool_bwd_kernel(const uint8_t* __restrict__ arg, const uint4* __restrict__ dy, uint4* __restrict__ dx,
                                   int64_t N, int H, int W, int OH, int OW, int CV) {
  // gather form: input pixel (iy, ix) sums dy of the (at most 4) windows whose recorded argmax tap is this pixel
  constexpr int V = Vec16<T>::N;
  const int64_t total = N * H * W * CV;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int cv = int(i % CV);
    int64_t t = i / CV;
    const int ix = int(t % W); t /= W;
    const int iy = int(t % H);
    const int64_t n = t / H;
    float g[V];
#pragma unroll
    for (int j = 0; j < V; ++j) g[j] = 0.0f;
    for (int oy = iy / 2; oy <= (iy + 1) / 2; ++oy) {
      if (oy >= OH) continue;
      const int kh = iy - (oy * 2 - 1);
      for (int ox = ix / 2; ox <= (ix + 1) / 2; ++ox) {
        if (ox >= OW) continue;
        const int kw = ix - (ox * 2 - 1);
        const uint8_t tap = uint8_t(kh * 3 + kw);
        const int64_t o = ((n * OH + oy) * OW + ox) * CV + cv;
        float d[V];
        Vec16<T>::unpack(__ldg(dy + o), d);
        const uint8_t* ap = arg + o * V;
#pragma unroll
        for (int j = 0; j < V; ++j)
          if (ap[j] == tap) g[j] += d[j];
      }
    }
    dx[i] = Vec16<T>::pack(g);
  }
}

template <typename T>
int maxpool3x3s2_fwd(const T* x, T* y, uint8_t* argmax, int64_t N, int H, int W, int C, cudaStream_t stream) {
  ProfScope prof("maxpool_fwd", stream);
  constexpr int V = Vec16<T>::N;
  TB_REQUIRE(C % V == 0, "maxpool: C must be a multiple of %d", V);
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  const int64_t total = N * OH * OW * (C / V);
  if (total == 0) return 0;
  maxpool_fwd_kernel<T><<<rgrid(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y),
                                                                argmax, N, H, W, OH, OW, C / V);
  return check_launch("maxpool_fwd_kernel");
}
template <typename T>
int maxpool3x3s2_bwd(const uint8_t* argmax, const T* dy, T* dx, int64_t N, int H, int W, int C, cudaStream_t stream) {
  ProfScope prof("maxpool_bwd", stream);
  constexpr int V = Vec16<T>::N;
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  const int64_t total = N * H * W * (C / V);
  if (total == 0) return 0;
  maxpool_bwd_kernel<T><<<rgrid(total, 256), 256, 0, stream>>>(argmax, reinterpret_cast<const uint4*>(dy),
                                                                reinterpret_cast<uint4*>(dx), N, H, W, OH, OW, C / V);
  return check_launch("maxpool_bwd_kernel");
}
template int maxpool3x3s2_fwd<float>(const float*, float*, uint8_t*, int64_t, int, int, int, cudaStream_t);
template int maxpool3x3s2_fwd<__nv_bfloat16>(const __nv_bfloat16*, __nv_bfloat16*, uint8_t*, int64_t, int, int, int, cudaStream_t);
template int maxpool3x3s2_bwd<float>(const uint8_t*, const float*, float*, int64_t, int, int, int, cudaStream_t);
template int maxpool3x3s2_bwd<__nv_bfloat16>(const uint8_t*, const __nv_bfloat16*, __nv_bfloat16*, int64_t, int, int, int,
                                             cudaStream_t);

template <typename T>
__global__ void relu_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int64_t nv) {
  constexpr int V = Vec16<T>::N;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
    float f[V];
    Vec16<T>::unpack(__ldg(x + i), f);
#pragma unroll
    for (int j = 0; j < V; ++j) f[j] = fmaxf(f[j], 0.0f);
    y[i] = Vec16<T>::pack(f);
  }
}
template <typename T>
__global__ void relu_bwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ dy, uint4* __restrict__ dx, int64_t nv) {
  constexpr int V = Vec16<T>::N;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
    float f[V], d[V];
    Vec16<T>::unpack(__ldg(x + i), f);
    Vec16<T>::unpack(__ldg(dy + i), d);
#pragma unroll
    for (int j = 0; j < V; ++j) d[j] = f[j] > 0.0f ? d[j] : 0.0f;
    dx[i] = Vec16<T>::pack(d);
  }
}
template <typename T>
int relu_fwd(const T* x, T* y, int64_t n, cudaStream_t stream) {
  ProfScope prof("relu_fwd", stream);
  constexpr int V = Vec16<T>::N;
  TB_REQUIRE(n % V == 0, "relu_fwd: size must be a multiple of %d", V);
  if (n == 0) return 0;
  relu_fwd_kernel<T><<<rgrid(n / V, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), n / V);
  return check_launch("relu_fwd_kernel");
}
template <typename T>
int relu_bwd(const T* x, const T* dy, T* dx, int64_t n, cudaStream_t stream) {
  ProfScope prof("relu_bwd", stream);
  constexpr int V = Vec16<T>::N;
  TB_REQUIRE(n % V == 0, "relu_bwd: size must be a multiple of %d", V);
  if (n == 0) return 0;
  relu_bwd_kernel<T><<<rgrid(n / V, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<const uint4*>(dy),
                                                             reinterpret_cast<uint4*>(dx), n / V);
  return check_launch("relu_bwd_kernel");
}
template int relu_fwd<float>(const float*, float*, int64_t, cudaStream_t);
template int relu_fwd<__nv_bfloat16>(const __nv_bfloat16*, __nv_bfloat16*, int64_t, cudaStream_t);
template int relu_bwd<float>(const float*, const float*, float*, int64_t, cudaStream_t);
template int relu_bwd<__nv_bfloat16>(const __nv_bfloat16*, const __nv_bfloat16*, __nv_bfloat16*, int64_t, cudaStream_t);

template <>
int colsum_t<float>(const float* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch, cudaStream_t stream) {
  return colsum(X, out, M, ncols, ld, scratch, stream);
}
template <>
int colsum_t<__nv_bfloat16>(const __nv_bfloat16* X, float* out, int64_t M, int64_t ncols, int64_t ld, float* scratch,
                            cudaStream_t stream) {
  return colsum_bf16(X, out, M, ncols, ld, scratch, stream);
}

__global__ void copy_f32_strided_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t rows, int64_t cols,
                                        int64_t ld, int64_t ldo) {
  const int64_t total = rows * ldo;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t r = i / ldo, c = i % ldo;
    out[i] = c < cols ? in[r * ld + c] : 0.0f;
  }
}
template <>
int convert_from_f32<float>(const float* in, float* out, int64_t rows, int64_t cols, int64_t ld, int64_t ldo, cudaStream_t stream) {
  if (rows * ldo == 0) return 0;
  copy_f32_strided_kernel<<<rgrid(rows * ldo, 256), 256, 0, stream>>>(in, out, rows, cols, ld, ldo);
  return check_launch("copy_f32_strided_kernel");
}
template <>
int convert_from_f32<__nv_bfloat16>(const float* in, __nv_bfloat16* out, int64_t rows, int64_t cols, int64_t ld, int64_t ldo,
                                    cudaStream_t stream) {
  return f32_to_bf16(in, out, rows, cols, ld, ldo, stream);
}

}  // namespace tb
