// Micro-benchmarks that size design decisions of the chain kernel (not product code):
//   1. issue rate of FFMA per SM, ILP 1..8;
//   2. period of back-to-back kernel nodes in a CUDA graph (empty kernel, and a kernel of
//      512 CTAs x 128 threads that spins ~5 us), i.e. the launch overhead a 10 us kernel pays;
//   3. the same with programmatic dependent launch edges (wait at the top: hides launch latency only);
//   4. a kernel whose CTAs have uneven durations (one in five spins three times as long, like the
//      chain kernel's Cholesky-round tail), plain and with PDL as the chain kernel uses it:
//      signal dependents at the top, wait just before the store, so that the next launch
//      fills the slots the short CTAs free.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench/ubench scripts/ubench/ubench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); return 1; } } while (0)

template <int ILP>
__global__ void ffma_kernel(float* out, int iters, float a, float b) {
  float acc[ILP];
#pragma unroll
  for (int i = 0; i < ILP; ++i) acc[i] = threadIdx.x * 1e-3f + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; ++i) acc[i] = fmaf(acc[i], a, b);
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < ILP; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void empty_kernel() {}
__global__ void spin_kernel(long long cycles, float* sink) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
  if (sink && threadIdx.x == 0 && blockIdx.x == 0) sink[0] = 1.f;
}
__global__ void spin_kernel_pdl(long long cycles, float* sink) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
  asm volatile("griddepcontrol.launch_dependents;");
  if (sink && threadIdx.x == 0 && blockIdx.x == 0) sink[0] = 1.f;
}

__global__ void spin_uneven_kernel(long long cycles, float* sink, int pdl) {
  if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const long long n = (blockIdx.x % 5 == 0) ? 3 * cycles : cycles;
  const long long t0 = clock64();
  while (clock64() - t0 < n) {}
  if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  if (threadIdx.x == 0) sink[blockIdx.x] = 1.f;
}

template <class F>
float time_ms(F f, int reps = 5) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  return best;
}

template <int ILP>
void run_fma(float* out, int sms, double ghz, int warps_per_sm) {
  const int iters = 4096;
  const int threads = 32 * warps_per_sm;  // one CTA per SM
  auto f1 = [&] { ffma_kernel<ILP><<<sms, threads>>>(out, iters, 1.0001f, 0.5f); };
  f1(); cudaDeviceSynchronize();
  const float m1 = time_ms(f1);
  const double inst = (double)iters * ILP * warps_per_sm;  // warp instructions per SM
  printf("warps/SM %2d ILP %d: FFMA %.3f warp-inst/clk/SM (%.1f fma/clk/SM)\n",
         warps_per_sm, ILP, inst / (m1 * 1e-3 * ghz * 1e9), 32 * inst / (m1 * 1e-3 * ghz * 1e9));
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const double ghz = khz * 1e-6;
  printf("%s, %d SMs, %.3f GHz (attribute)\n", p.name, p.multiProcessorCount, ghz);
  float* out; CK(cudaMalloc(&out, 1 << 24));
  for (int w : {4, 8, 16, 32}) {
    run_fma<1>(out, p.multiProcessorCount, ghz, w);
    run_fma<2>(out, p.multiProcessorCount, ghz, w);
    run_fma<4>(out, p.multiProcessorCount, ghz, w);
    run_fma<8>(out, p.multiProcessorCount, ghz, w);
  }
  // graph of N kernel nodes: period per node
  cudaStream_t s; CK(cudaStreamCreate(&s));
  const int N = 200;
  for (int variant = 0; variant < 6; ++variant) {
    cudaGraph_t g; cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    for (int i = 0; i < N; ++i) {
      if (variant == 0) empty_kernel<<<1, 32, 0, s>>>();
      else if (variant == 1) empty_kernel<<<512, 128, 0, s>>>();
      else if (variant == 2) spin_kernel<<<512, 128, 0, s>>>(10000, out);
      else if (variant == 4) spin_uneven_kernel<<<512, 128, 0, s>>>(10000, out, 0);
      else {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(512); cfg.blockDim = dim3(128); cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (variant == 3) CK(cudaLaunchKernelEx(&cfg, spin_kernel_pdl, (long long)10000, out));
        else CK(cudaLaunchKernelEx(&cfg, spin_uneven_kernel, (long long)10000, out, 1));
      }
    }
    CK(cudaStreamEndCapture(s, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    CK(cudaGraphLaunch(ge, s)); CK(cudaStreamSynchronize(s));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e30f;
    for (int r = 0; r < 5; ++r) {
      cudaEventRecord(e0, s); cudaGraphLaunch(ge, s); cudaEventRecord(e1, s); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    const char* names[] = {"empty <<<1,32>>>", "empty <<<512,128>>>", "spin 10000 clk <<<512,128>>>",
                           "spin 10000 clk <<<512,128>>> + PDL (wait at the top)",
                           "uneven spin 10000 / 30000 clk <<<512,128>>>",
                           "uneven spin 10000 / 30000 clk <<<512,128>>> + PDL (signal at the top, wait before the store)"};
    printf("graph of %d nodes, %s: %.2f us per node\n", N, names[variant], best * 1e3 / N);
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  }
  return 0;
}
