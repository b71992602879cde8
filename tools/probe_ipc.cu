// Feasibility probe for the peer-memory ring transport (DESIGN.md §3.5): N forked processes, one GPU each,
// exchange cudaIpc handles of a heap, then measure
//   A  copy-engine PULL bandwidth from a peer's heap (cudaMemcpyAsync on a peer-mapped pointer), all ranks at once
//   B  the same while a spinning kernel occupies every SM (the attention kernels leave no SM free)
//   C  three ways of raising a 32-bit flag in a PEER's heap + cuStreamWaitValue32 on the local flag (ping-pong latency)
//   D  put-then-signal ordering (payload visible once the flag is)
// usage: probe_ipc [n_gpus=2]
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <sys/mman.h>
#include <sys/wait.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("[r%d] %s:%d %s -> %s\n", g_rank, __FILE__, __LINE__, #x, cudaGetErrorString(e_)); fflush(stdout); exit(2); } } while (0)

static int g_rank = -1;

struct Shared {
  cudaIpcMemHandle_t handles[8];
  volatile int arrive[64];
};

static void host_barrier(Shared* sh, int n, int* phase) {
  const int p = (*phase)++;
  __sync_fetch_and_add(&sh->arrive[p], 1);
  while (sh->arrive[p] < n) usleep(50);
}

__global__ void spin_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}
__global__ void fill_kernel(unsigned* p, size_t n, unsigned v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void check_kernel(const unsigned* p, size_t n, unsigned v, unsigned* bad) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    if (p[i] != v) atomicAdd(bad, 1u);
}

typedef CUresult (*wait32_t)(CUstream, CUdeviceptr, cuuint32_t, unsigned);
typedef CUresult (*write32_t)(CUstream, CUdeviceptr, cuuint32_t, unsigned);
typedef CUresult (*memset32_t)(CUdeviceptr, unsigned, size_t, CUstream);

static void* drv(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
    printf("[r%d] driver entry point %s not found\n", g_rank, name);
    return nullptr;
  }
  return fn;
}

int main(int argc, char** argv) {
  const int n = argc > 1 ? atoi(argv[1]) : 2;
  Shared* sh = (Shared*)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  memset(sh, 0, sizeof(Shared));
  for (int r = 0; r < n; ++r) {
    pid_t pid = fork();
    if (pid == 0) { g_rank = r; break; }
  }
  if (g_rank < 0) {
    int st, rc = 0;
    while (wait(&st) > 0) rc |= st;
    return rc ? 1 : 0;
  }
  const int r = g_rank;
  int phase = 0;
  CK(cudaSetDevice(r));
  const size_t kFlagBytes = 1 << 16, kData = size_t(256) << 20;
  unsigned char* heap = nullptr;
  CK(cudaMalloc(&heap, kFlagBytes + 2 * kData));
  CK(cudaMemset(heap, 0, kFlagBytes));
  CK(cudaIpcGetMemHandle(&sh->handles[r], heap));
  host_barrier(sh, n, &phase);
  unsigned char* peer_heap[8];
  for (int p = 0; p < n; ++p) {
    if (p == r) { peer_heap[p] = heap; continue; }
    CK(cudaIpcOpenMemHandle((void**)&peer_heap[p], sh->handles[p], cudaIpcMemLazyEnablePeerAccess));
  }
  if (r == 0) printf("ipc: %d ranks mapped each other's heaps\n", n);
  cudaStream_t s_copy, s_main;
  CK(cudaStreamCreateWithFlags(&s_copy, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s_main, cudaStreamNonBlocking));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  unsigned* data = (unsigned*)(heap + kFlagBytes);
  unsigned* land = (unsigned*)(heap + kFlagBytes + kData);
  fill_kernel<<<296, 1024, 0, s_main>>>(data, kData / 4, 0x1000u + r);
  CK(cudaStreamSynchronize(s_main));
  host_barrier(sh, n, &phase);
  const int src = (r + 1) % n;
  // ---- A / B: pull bandwidth
  for (int busy = 0; busy < 2; ++busy) {
    for (int it = 0; it < 3; ++it) {
      host_barrier(sh, n, &phase);
      if (busy) spin_kernel<<<132 * 2, 1024, 0, s_main>>>(100000000LL);   // ~50 ms, every SM fully occupied
      CK(cudaEventRecord(e0, s_copy));
      CK(cudaMemcpyAsync(land, peer_heap[src] + kFlagBytes, kData, cudaMemcpyDeviceToDevice, s_copy));
      CK(cudaEventRecord(e1, s_copy));
      CK(cudaStreamSynchronize(s_copy));
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (it == 2) printf("[r%d] pull 256 MiB from r%d %s: %.3f ms = %.0f GB/s\n", r, src, busy ? "(SMs busy)" : "(idle)  ", ms, kData / ms / 1e6);
      CK(cudaStreamSynchronize(s_main));
    }
  }
  unsigned* bad = nullptr;
  CK(cudaMalloc(&bad, 4));
  CK(cudaMemset(bad, 0, 4));
  check_kernel<<<296, 1024, 0, s_main>>>(land, kData / 4, 0x1000u + src, bad);
  unsigned hb = 1;
  CK(cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost));
  printf("[r%d] pulled payload %s\n", r, hb ? "CORRUPT" : "ok");
  // small pulls (latency)
  for (size_t bytes : {size_t(4096), size_t(1) << 20, size_t(16) << 20, size_t(64) << 20}) {
    host_barrier(sh, n, &phase);
    CK(cudaEventRecord(e0, s_copy));
    for (int i = 0; i < 8; ++i)
      CK(cudaMemcpyAsync((char*)land + i * bytes % kData, peer_heap[src] + kFlagBytes + i * bytes % kData, bytes, cudaMemcpyDeviceToDevice, s_copy));
    CK(cudaEventRecord(e1, s_copy));
    CK(cudaStreamSynchronize(s_copy));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (r == 0) printf("[r0] 8 pulls of %zu KiB: %.1f us each, %.0f GB/s\n", bytes >> 10, ms * 1e3 / 8, 8 * bytes / ms / 1e6);
  }

  // ---- C: flags. slot layout in every heap: flags[method][writer_rank]
  wait32_t f_wait = (wait32_t)drv("cuStreamWaitValue32");
  write32_t f_write = (write32_t)drv("cuStreamWriteValue32");
  memset32_t f_memset = (memset32_t)drv("cuMemsetD32Async");
  unsigned* vals = nullptr;   // table of constants for the 4-byte memcpy signal
  CK(cudaMalloc(&vals, 4096 * 4));
  {
    unsigned h[4096];
    for (int i = 0; i < 4096; ++i) h[i] = i;
    CK(cudaMemcpy(vals, h, sizeof(h), cudaMemcpyHostToDevice));
  }
  const int peer = r ^ 1;
  if (peer < n && f_wait) {
    for (int m = 0; m < 3; ++m) {
      const char* mname[3] = {"cuStreamWriteValue32(peer ptr)", "cuMemsetD32Async(peer ptr)", "4-byte cudaMemcpyAsync"};
      unsigned* my_flag = (unsigned*)heap + m * 16 + peer;                   // written by `peer`
      unsigned* peer_flag = (unsigned*)peer_heap[peer] + m * 16 + r;         // I write it
      host_barrier(sh, n, &phase);
      CUresult cr = CUDA_SUCCESS;
      const int rounds = 200;
      CK(cudaEventRecord(e0, s_copy));
      for (int i = 1; i <= rounds && cr == CUDA_SUCCESS; ++i) {
        // ping-pong: even rank signals first
        for (int half = 0; half < 2 && cr == CUDA_SUCCESS; ++half) {
          const bool my_turn = ((r & 1) == half);
          if (my_turn) {
            if (m == 0) cr = f_write ? f_write((CUstream)s_copy, (CUdeviceptr)peer_flag, i, 0) : CUDA_ERROR_NOT_FOUND;
            else if (m == 1) cr = f_memset ? f_memset((CUdeviceptr)peer_flag, i, 1, (CUstream)s_copy) : CUDA_ERROR_NOT_FOUND;
            else cr = (CUresult)cudaMemcpyAsync(peer_flag, vals + i, 4, cudaMemcpyDeviceToDevice, s_copy);
          } else {
            cr = f_wait((CUstream)s_copy, (CUdeviceptr)my_flag, i, CU_STREAM_WAIT_VALUE_GEQ);
          }
        }
      }
      if (cr != CUDA_SUCCESS) {
        printf("[r%d] flag method %d %s: FAILED to enqueue (CUresult %d)\n", r, m, mname[m], (int)cr);
        cudaGetLastError();
        // release a peer that may be waiting: fall back to memcpy writes of the final value
        cudaMemcpyAsync(peer_flag, vals + rounds, 4, cudaMemcpyDeviceToDevice, s_main);
        cudaStreamSynchronize(s_main);
      }
      CK(cudaEventRecord(e1, s_copy));
      cudaError_t se = cudaStreamSynchronize(s_copy);
      float ms = 0;
      if (se == cudaSuccess) CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("[r%d] flag method %d %-32s: %s, %.1f us per round trip\n", r, m, mname[m],
             se == cudaSuccess && cr == CUDA_SUCCESS ? "ok" : cudaGetErrorString(se), ms * 1e3 / rounds);
      if (se != cudaSuccess) exit(3);
    }
    // ---- D: put 64 MiB then signal (method 2, always valid); the receiver waits on the flag, then checks the payload
    for (int m : {0, 2}) {
      if (m == 0 && !f_write) continue;
      host_barrier(sh, n, &phase);
      unsigned* my_flag = (unsigned*)heap + (8 + m) * 16 + peer;
      unsigned* peer_flag = (unsigned*)peer_heap[peer] + (8 + m) * 16 + r;
      const size_t bytes = size_t(64) << 20;
      fill_kernel<<<296, 1024, 0, s_copy>>>(data, bytes / 4, 0xabc00000u + m * 16 + r);
      CK(cudaMemcpyAsync(peer_heap[peer] + kFlagBytes + kData, data, bytes, cudaMemcpyDeviceToDevice, s_copy));   // PUT into peer's landing
      if (m == 0) f_write((CUstream)s_copy, (CUdeviceptr)peer_flag, 7, 0);
      else CK(cudaMemcpyAsync(peer_flag, vals + 7, 4, cudaMemcpyDeviceToDevice, s_copy));
      f_wait((CUstream)s_main, (CUdeviceptr)my_flag, 7, CU_STREAM_WAIT_VALUE_GEQ);
      CK(cudaMemsetAsync(bad, 0, 4, s_main));
      check_kernel<<<296, 1024, 0, s_main>>>(land, bytes / 4, 0xabc00000u + m * 16 + peer, bad);
      CK(cudaMemcpyAsync(&hb, bad, 4, cudaMemcpyDeviceToHost, s_main));
      CK(cudaStreamSynchronize(s_main));
      CK(cudaStreamSynchronize(s_copy));
      printf("[r%d] put-then-signal (method %d): payload %s\n", r, m, hb ? "NOT VISIBLE / corrupt" : "visible and correct");
    }
  }
  host_barrier(sh, n, &phase);
  for (int p = 0; p < n; ++p)
    if (p != r) CK(cudaIpcCloseMemHandle(peer_heap[p]));
  host_barrier(sh, n, &phase);
  CK(cudaFree(heap));
  if (r == 0) printf("probe_ipc done\n");
  return 0;
}
