// Micro-benchmark: FP64 throughput of one SM pipe via DFMA vs mma.sync.m8n8k4.f64 (DMMA).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_pipes fp64_pipes.cu && ./fp64_pipes
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_dfma(double *out, int iters)
{
    double a[8], b = 1.000001, c = 0.5;
    for (int i = 0; i < 8; i++) a[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++)
#pragma unroll
        for (int i = 0; i < 8; i++) a[i] = fma(a[i], b, c);
    double s = 0;
    for (int i = 0; i < 8; i++) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma(double *out, int iters)
{
    double c[8][2];
    for (int i = 0; i < 8; i++) c[i][0] = c[i][1] = 0.0;
    double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
    for (int it = 0; it < iters; it++)
#pragma unroll
        for (int i = 0; i < 8; i++)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
    double s = 0;
    for (int i = 0; i < 8; i++) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main()
{
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    double *out;
    cudaMalloc(&out, sizeof(double) * 1024 * 1024);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int iters = 20000;
    for (int threads : {128, 256, 512, 1024}) {
        float ms;
        k_dfma<<<sms, threads>>>(out, 100);
        cudaEventRecord(e0); k_dfma<<<sms, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        double fl = 2.0 * 8 * iters * (double) threads * sms;
        printf("DFMA  %4d thr/SM: %.2f TFLOP/s\n", threads, fl / ms * 1e-9);
        k_dmma<<<sms, threads>>>(out, 100);
        cudaEventRecord(e0); k_dmma<<<sms, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        fl = 2.0 * 8 * 8 * 4 * 8 * iters * (double) (threads / 32) * sms; // 8 mma of 8x8x4 per iter per warp
        printf("DMMA  %4d thr/SM: %.2f TFLOP/s\n", threads, fl / ms * 1e-9);
    }
    printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
