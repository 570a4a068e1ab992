// Probe used for DESIGN.md section 4 (launch policy): nvcc -O2 -gencode arch=compute_90a,code=sm_90a -o smid_probe scripts/smid_probe.cu
// prints how many blocks of two concurrent kernels each SM received.
// how does the block scheduler spread two concurrent kernels over the SMs?
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>
__global__ void k(int* smid_out, long long spin) {
    extern __shared__ unsigned char sm[];
    unsigned s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
    if (threadIdx.x == 0) smid_out[blockIdx.x] = (int)s;
    long long t0 = clock64();
    while (clock64() - t0 < spin) { sm[threadIdx.x] += 1; }
}
int main(int argc, char** argv) {
    int nA = argc > 1 ? atoi(argv[1]) : 569, thA = argc > 2 ? atoi(argv[2]) : 64, smA = argc > 3 ? atoi(argv[3]) : 27000;
    int nB = argc > 4 ? atoi(argv[4]) : 440, thB = argc > 5 ? atoi(argv[5]) : 128, smB = argc > 6 ? atoi(argv[6]) : 63800;
    int *a, *b; cudaMalloc(&a, nA * 4); cudaMalloc(&b, nB * 4);
    cudaMemset(a, 0xff, nA * 4); cudaMemset(b, 0xff, nB * 4);
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200000);
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaStream_t s1, s2; cudaStreamCreate(&s1); cudaStreamCreate(&s2);
    k<<<nA, thA, smA, s1>>>(a, 2000000);
    k<<<nB, thB, smB, s2>>>(b, 2000000);
    cudaDeviceSynchronize();
    std::vector<int> ha(nA), hb(nB); cudaMemcpy(ha.data(), a, nA * 4, cudaMemcpyDeviceToHost); cudaMemcpy(hb.data(), b, nB * 4, cudaMemcpyDeviceToHost);
    int ca[160] = {0}, cb[160] = {0};
    for (int x : ha) if (x >= 0 && x < 160) ca[x]++;
    for (int x : hb) if (x >= 0 && x < 160) cb[x]++;
    printf("per-SM (A,B) block counts over the whole run:\n");
    int n_sm = 0; cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
    for (int i = 0; i < n_sm && i < 160; ++i) printf("%d:%d,%d ", i, ca[i], cb[i]);
    printf("\nfirst 20 A blocks -> SM: "); for (int i = 0; i < 20; ++i) printf("%d ", ha[i]);
    printf("\n");
    return 0;
}
