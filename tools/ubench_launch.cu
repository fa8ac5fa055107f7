// ubench_launch.cu — launch / barrier / graph overheads on the GPU box (decides how the `fast` frame is driven).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o ubench_launch ubench_launch.cu && ./ubench_launch
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("ERR %s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); return 1; } } while (0)

__global__ void k_empty(int* p) { if (p && threadIdx.x == 0 && blockIdx.x == 0x7fffffff) *p = 1; }
__global__ void k_touch(int* p, int n) { const int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] += 1; }

__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    while (((volatile unsigned int*)bar)[0] < target) {}
    __threadfence();
  }
  __syncthreads();
}
__global__ void k_barrier_loop(unsigned int* bar, int iters, int* sink) {
  unsigned int epoch = 0;
  for (int i = 0; i < iters; ++i) grid_barrier(bar, (++epoch) * gridDim.x);
  if (sink && blockIdx.x == 0 && threadIdx.x == 0) *sink = (int)epoch;
}
__global__ void k_cg_barrier_loop(int iters, int* sink) {
  cooperative_groups::grid_group g = cooperative_groups::this_grid();
  for (int i = 0; i < iters; ++i) g.sync();
  if (sink && blockIdx.x == 0 && threadIdx.x == 0) *sink = iters;
}

__global__ void k_while_body(int* counter, cudaGraphConditionalHandle h) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int c = --(*counter);
    cudaGraphSetConditional(h, c > 0 ? 1u : 0u);
  }
}
__global__ void k_set_counter(int* counter, int v, cudaGraphConditionalHandle h) { *counter = v; cudaGraphSetConditional(h, 1u); }

static float elapsed(cudaEvent_t a, cudaEvent_t b) { float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }

int main() {
  setvbuf(stdout, nullptr, _IONBF, 0);
  cudaStream_t s;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  int* d = nullptr;
  CK(cudaMalloc(&d, 4 << 20));
  CK(cudaMemset(d, 0, 4 << 20));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sm = prop.multiProcessorCount;
  printf("device %s, %d SMs\n", prop.name, sm);

  // 1. stream launches, host running ahead
  for (int rep = 0; rep < 2; ++rep) {
    const int N = 2000;
    CK(cudaEventRecord(e0, s));
    for (int i = 0; i < N; ++i) k_empty<<<1, 32, 0, s>>>(d);
    CK(cudaEventRecord(e1, s));
    CK(cudaStreamSynchronize(s));
    if (rep) printf("stream launch, empty <<<1,32>>>      : %.3f us / kernel\n", 1e3 * elapsed(e0, e1) / N);
  }
  for (int rep = 0; rep < 2; ++rep) {
    const int N = 2000;
    CK(cudaEventRecord(e0, s));
    for (int i = 0; i < N; ++i) k_touch<<<sm * 8, 256, 0, s>>>(d, sm * 8 * 256);
    CK(cudaEventRecord(e1, s));
    CK(cudaStreamSynchronize(s));
    if (rep) printf("stream launch, touch <<<%d,256>>>   : %.3f us / kernel\n", sm * 8, 1e3 * elapsed(e0, e1) / N);
  }
  // 1b. launch + sync round trip (what a host read-back costs)
  {
    const int N = 500;
    int* h = nullptr;
    CK(cudaMallocHost(&h, 256));
    CK(cudaStreamSynchronize(s));
    cudaEvent_t w0, w1;
    cudaEventCreate(&w0); cudaEventCreate(&w1);
    CK(cudaEventRecord(e0, s));
    for (int i = 0; i < N; ++i) {
      k_empty<<<1, 32, 0, s>>>(d);
      CK(cudaMemcpyAsync(h, d, 152, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
    }
    CK(cudaEventRecord(e1, s));
    CK(cudaStreamSynchronize(s));
    printf("kernel + 152 B D2H + stream sync      : %.3f us / round trip\n", 1e3 * elapsed(e0, e1) / N);
  }
  // 2. graph of 30 chained kernels
  for (int big = 0; big < 2; ++big) {
    cudaGraph_t g;
    cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal));
    for (int i = 0; i < 30; ++i) { if (big) k_touch<<<sm * 8, 256, 0, s>>>(d, sm * 8 * 256); else k_empty<<<1, 32, 0, s>>>(d); }
    CK(cudaStreamEndCapture(s, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    for (int rep = 0; rep < 2; ++rep) {
      const int N = 200;
      CK(cudaEventRecord(e0, s));
      for (int i = 0; i < N; ++i) CK(cudaGraphLaunch(ge, s));
      CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      if (rep) printf("graph of 30 chained %s kernels     : %.3f us / kernel (%.1f us / graph)\n", big ? "touch" : "empty", 1e3 * elapsed(e0, e1) / N / 30, 1e3 * elapsed(e0, e1) / N);
    }
    // graph launch + sync per graph (frame-synchronous API)
    {
      const int N = 200;
      CK(cudaEventRecord(e0, s));
      for (int i = 0; i < N; ++i) { CK(cudaGraphLaunch(ge, s)); CK(cudaStreamSynchronize(s)); }
      CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      printf("  same, one stream sync per graph     : %.1f us / graph\n", 1e3 * elapsed(e0, e1) / N);
    }
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  }
  // 3. grid barriers in a persistent kernel
  {
    unsigned int* bar = nullptr;
    CK(cudaMalloc(&bar, 256));
    const int cfgs[4][2] = {{1, 256}, {1, 1024}, {2, 512}, {4, 256}};
    for (auto& c : cfgs) {
      const int grid = sm * c[0], threads = c[1], iters = 2000;
      CK(cudaMemsetAsync(bar, 0, 4, s));
      void* args[] = {(void*)&bar, (void*)&iters, (void*)&d};
      CK(cudaEventRecord(e0, s));
      CK(cudaLaunchCooperativeKernel((const void*)k_barrier_loop, dim3(grid), dim3(threads), args, 0, s));
      CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      printf("grid barrier (atomic+spin) %4d x %4d : %.3f us / barrier\n", grid, threads, 1e3 * elapsed(e0, e1) / iters);
      void* args2[] = {(void*)&iters, (void*)&d};
      CK(cudaEventRecord(e0, s));
      CK(cudaLaunchCooperativeKernel((const void*)k_cg_barrier_loop, dim3(grid), dim3(threads), args2, 0, s));
      CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      printf("grid barrier (cg grid.sync) %4d x %4d: %.3f us / barrier\n", grid, threads, 1e3 * elapsed(e0, e1) / iters);
    }
  }
  // 4. conditional WHILE node: per-iteration overhead
  {
    cudaGraph_t g;
    CK(cudaGraphCreate(&g, 0));
    cudaGraphConditionalHandle h;
    CK(cudaGraphConditionalHandleCreate(&h, g, 0, 0));
    int* counter = d + 1024;
    // node A: set counter
    cudaGraphNode_t nA;
    int iters = 100;
    {
      cudaKernelNodeParams kp = {};
      void* args[] = {(void*)&counter, (void*)&iters, (void*)&h};
      kp.func = (void*)k_set_counter; kp.gridDim = dim3(1); kp.blockDim = dim3(1); kp.kernelParams = args;
      CK(cudaGraphAddKernelNode(&nA, g, nullptr, 0, &kp));
    }
    cudaGraphNode_t nW;
    cudaGraphNodeParams cp = {};
    cp.type = cudaGraphNodeTypeConditional;
    cp.conditional.handle = h;
    cp.conditional.type = cudaGraphCondTypeWhile;
    cp.conditional.size = 1;
    CK(cudaGraphAddNode(&nW, g, &nA, 1, &cp));
    cudaGraph_t body = cp.conditional.phGraph_out[0];
    {
      cudaGraphNode_t nB, nC;
      cudaKernelNodeParams kp = {};
      int n = sm * 8 * 256;
      void* args0[] = {(void*)&d, (void*)&n};
      kp.func = (void*)k_touch; kp.gridDim = dim3(sm * 8); kp.blockDim = dim3(256); kp.kernelParams = args0;
      CK(cudaGraphAddKernelNode(&nC, body, nullptr, 0, &kp));
      void* args[] = {(void*)&counter, (void*)&h};
      kp.func = (void*)k_while_body; kp.gridDim = dim3(1); kp.blockDim = dim3(32); kp.kernelParams = args;
      CK(cudaGraphAddKernelNode(&nB, body, &nC, 1, &kp));
    }
    cudaGraphExec_t ge;
    CK(cudaGraphInstantiate(&ge, g, 0));
    for (int rep = 0; rep < 2; ++rep) {
      const int N = 50;
      CK(cudaEventRecord(e0, s));
      for (int i = 0; i < N; ++i) CK(cudaGraphLaunch(ge, s));
      CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      if (rep) printf("conditional WHILE node, body = touch + cond kernel: %.3f us / iteration (100 iterations / graph)\n", 1e3 * elapsed(e0, e1) / N / 100);
    }
  }
  // 5. memset node cost: 25 MB of clears per frame today
  {
    const int N = 200;
    uint8_t* big = nullptr;
    CK(cudaMalloc(&big, 32 << 20));
    CK(cudaEventRecord(e0, s));
    for (int i = 0; i < N; ++i) { cudaMemsetAsync(big, 0xFF, 16 << 20, s); cudaMemsetAsync(big + (16 << 20), 0, 5 << 20, s); cudaMemsetAsync(big + (24 << 20), 0x7F, 4 << 20, s); }
    CK(cudaEventRecord(e1, s));
    CK(cudaStreamSynchronize(s));
    printf("3 memsets (16 + 5 + 4 MB)             : %.3f us / frame\n", 1e3 * elapsed(e0, e1) / N);
  }
  printf("done\n");
  return 0;
}
