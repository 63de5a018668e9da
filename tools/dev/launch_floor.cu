// Launch floors for tools/dev/launch_gap.py: an empty kernel with the solo solve's launch shape (one 1024-thread block
// per SM, the fused kernel's 43 744 B of static shared memory plus the same dynamic shared memory, an 832-byte
// argument struct), timed with CUDA events on an idle stream three ways:
//   0  a one-node graph whose kernel parameters are patched (cudaGraphExecKernelNodeSetParams) before each launch;
//   1  the same with an external event-wait node in front, on an event recorded just before on a second, idle stream;
//   2  a direct cudaLaunchKernelEx.
// Built by launch_gap.py with nvcc into a temporary directory; loaded with ctypes.
#include <cuda_runtime.h>

namespace {

struct FloorArgs {
  unsigned char b[832];  // sizeof(yd::FusedArgs)
};

__global__ void __launch_bounds__(1024, 1) k_floor(FloorArgs a) {
  __shared__ unsigned pad[43744 / 4];  // k_fused_front's static shared memory: the same carveout
  extern __shared__ unsigned dyn[];
  if (a.b[0] == 0xAB) {  // never true: keeps both arrays without touching them
    pad[threadIdx.x] = threadIdx.x;
    __syncthreads();
    dyn[threadIdx.x] = pad[1023 - threadIdx.x];
  }
}

cudaStream_t g_st = nullptr, g_side = nullptr;
cudaEvent_t g_ev1 = nullptr, g_ev4 = nullptr, g_dep = nullptr;
cudaGraph_t g_graph[2] = {};  // kept: their kernel nodes name the nodes to patch in the instantiated graphs
cudaGraphExec_t g_exec[2] = {};
cudaGraphNode_t g_node[2] = {};
FloorArgs g_args{};
unsigned g_grid = 0;
size_t g_dyn = 0;

cudaError_t g_err = cudaSuccess;

#define FLOOR_CHECK(x) do { if ((g_err = (x)) != cudaSuccess) return -1; } while (0)

int Capture(int i) {
  cudaGraph_t& graph = g_graph[i];
  FLOOR_CHECK(cudaStreamBeginCapture(g_st, cudaStreamCaptureModeThreadLocal));
  if (i == 1) FLOOR_CHECK(cudaStreamWaitEvent(g_st, g_dep, cudaEventWaitExternal));
  k_floor<<<g_grid, 1024, g_dyn, g_st>>>(g_args);
  FLOOR_CHECK(cudaStreamEndCapture(g_st, &graph));
  FLOOR_CHECK(cudaGraphInstantiate(&g_exec[i], graph, 0));
  size_t n = 0;
  FLOOR_CHECK(cudaGraphGetNodes(graph, nullptr, &n));
  cudaGraphNode_t nodes[2];
  if (n > 2) return -1;
  FLOOR_CHECK(cudaGraphGetNodes(graph, nodes, &n));
  for (size_t k = 0; k != n; ++k) {
    cudaGraphNodeType ty;
    FLOOR_CHECK(cudaGraphNodeGetType(nodes[k], &ty));
    if (ty == cudaGraphNodeTypeKernel) g_node[i] = nodes[k];
  }
  return g_node[i] ? 0 : -1;
}

}  // namespace

extern "C" int floor_init(unsigned grid, size_t dyn) {
  g_grid = grid;
  g_dyn = dyn;
  FLOOR_CHECK(cudaFuncSetAttribute(k_floor, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
  FLOOR_CHECK(cudaStreamCreateWithFlags(&g_st, cudaStreamNonBlocking));
  FLOOR_CHECK(cudaStreamCreateWithFlags(&g_side, cudaStreamNonBlocking));
  FLOOR_CHECK(cudaEventCreate(&g_ev1));
  FLOOR_CHECK(cudaEventCreate(&g_ev4));
  FLOOR_CHECK(cudaEventCreateWithFlags(&g_dep, cudaEventDisableTiming));
  FLOOR_CHECK(cudaEventRecord(g_dep, g_side));
  if (Capture(0) || Capture(1)) return -1;
  return 0;
}

// One launch of the given kind between two events; milliseconds, or < 0 on an error.
extern "C" float floor_once(int mode) {
  g_args.b[1] += 1;  // new arguments every call, as a solve's scalars
  if (mode == 0 || mode == 1) {
    if (mode == 1) FLOOR_CHECK(cudaEventRecord(g_dep, g_side));
    void* kp[1] = {&g_args};
    cudaKernelNodeParams np{};
    np.func = reinterpret_cast<void*>(k_floor);
    np.gridDim = dim3(g_grid);
    np.blockDim = dim3(1024);
    np.sharedMemBytes = (unsigned)g_dyn;
    np.kernelParams = kp;
    FLOOR_CHECK(cudaGraphExecKernelNodeSetParams(g_exec[mode], g_node[mode], &np));
    FLOOR_CHECK(cudaEventRecord(g_ev1, g_st));
    FLOOR_CHECK(cudaGraphLaunch(g_exec[mode], g_st));
    FLOOR_CHECK(cudaEventRecord(g_ev4, g_st));
  } else {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(g_grid);
    cfg.blockDim = dim3(1024);
    cfg.dynamicSmemBytes = g_dyn;
    cfg.stream = g_st;
    FLOOR_CHECK(cudaEventRecord(g_ev1, g_st));
    FLOOR_CHECK(cudaLaunchKernelEx(&cfg, k_floor, g_args));
    FLOOR_CHECK(cudaEventRecord(g_ev4, g_st));
  }
  FLOOR_CHECK(cudaStreamSynchronize(g_st));
  float ms = 0;
  FLOOR_CHECK(cudaEventElapsedTime(&ms, g_ev1, g_ev4));
  return ms;
}

// The error of the call that failed last.
extern "C" const char* floor_error() { return cudaGetErrorString(g_err); }

extern "C" void floor_close() {
  for (auto& e : g_exec) if (e) cudaGraphExecDestroy(e);
  for (auto& g : g_graph) if (g) cudaGraphDestroy(g);
  cudaEventDestroy(g_ev1);
  cudaEventDestroy(g_ev4);
  cudaEventDestroy(g_dep);
  cudaStreamDestroy(g_st);
  cudaStreamDestroy(g_side);
}
