// Microbenchmark: peak DMMA rate per SM on the attached GPU for the f64 mma.sync shapes m8n8k4 (the reference instances
// of the GEMM kernels) and m16n8k4 (the shape the GEMM kernels issue) / m16n8k16 (sm_90), and the plain DFMA rate.
// Not part of the product.
#include <cstdio>
#include <cuda_runtime.h>

template <int NACC>
__global__ void dmma_kernel(double* out, int iters, double a0, double b0) {
    double acc[NACC][2];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i][0] = acc[i][1] = 0.0;
    double a = a0 + threadIdx.x, b = b0 + threadIdx.x;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(acc[i][0]), "+d"(acc[i][1]) : "d"(a), "d"(b));
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; ++i) s += acc[i][0] + acc[i][1];
    if (s == 123.456) out[0] = s;
}

// m16n8k4: A 2, B 1, C/D 4 doubles per lane (512 FMA per warp instruction); m16n8k16: A 8, B 4, C/D 4 (2048 FMA)
template <int NACC, int K>
__global__ void dmma16_kernel(double* out, int iters, double a0, double b0) {
    double acc[NACC][4];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.0;
    double a = a0 + threadIdx.x, b = b0 + threadIdx.x;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
            if (K == 4)
                asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4}, {%5}, {%0,%1,%2,%3};"
                             : "+d"(acc[i][0]), "+d"(acc[i][1]), "+d"(acc[i][2]), "+d"(acc[i][3]) : "d"(a), "d"(b));
            else
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4,%4,%4,%4,%4,%4,%4}, "
                             "{%5,%5,%5,%5}, {%0,%1,%2,%3};"
                             : "+d"(acc[i][0]), "+d"(acc[i][1]), "+d"(acc[i][2]), "+d"(acc[i][3]) : "d"(a), "d"(b));
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; ++i) s += acc[i][0] + acc[i][1] + acc[i][2] + acc[i][3];
    if (s == 123.456) out[0] = s;
}

template <int NACC>
__global__ void dfma_kernel(double* out, int iters, double a0, double b0) {
    double acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = i;
    double a = a0 + threadIdx.x, b = b0;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = fma(acc[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < NACC; ++i) s += acc[i];
    if (s == 123.456) out[0] = s;
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    printf("device %s sms %d clock %d kHz\n", p.name, sms, p.clockRate);
    double* out;
    cudaMalloc(&out, 8);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    const int iters = 20000;
    for (int warps : {1, 2, 4, 8, 16}) {
        for (int rep = 0; rep < 2; ++rep) {
            cudaEventRecord(e0);
            dmma_kernel<16><<<sms, warps * 32>>>(out, iters, 1.0, 2.0);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms;
            cudaEventElapsedTime(&ms, e0, e1);
            double fma = (double)sms * warps * iters * 16 * 256.0;
            if (rep) printf("DMMA warps/SM %2d: %.3f ms  %.2f TFLOP/s  (%.1f FMA/ns/SM)\n", warps, ms, 2 * fma / ms / 1e9, fma / ms / 1e6 / sms);
        }
    }
    for (int k : {4, 16}) {
        for (int warps : {4, 8, 16}) {
            for (int rep = 0; rep < 2; ++rep) {
                const int it = k == 4 ? iters : iters / 4;
                cudaEventRecord(e0);
                if (k == 4) dmma16_kernel<8, 4><<<sms, warps * 32>>>(out, it, 1.0, 2.0);
                else dmma16_kernel<8, 16><<<sms, warps * 32>>>(out, it, 1.0, 2.0);
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                float ms;
                cudaEventElapsedTime(&ms, e0, e1);
                double fma = (double)sms * warps * it * 8 * (16.0 * 8 * k);
                if (rep) printf("DMMA m16n8k%d warps/SM %2d: %.3f ms  %.2f TFLOP/s  (%.1f FMA/ns/SM)\n", k, warps, ms, 2 * fma / ms / 1e9,
                                fma / ms / 1e6 / sms);
            }
        }
    }
    for (int warps : {4, 8, 16, 32}) {
        for (int rep = 0; rep < 2; ++rep) {
            cudaEventRecord(e0);
            dfma_kernel<16><<<sms, warps * 32>>>(out, iters, 1.0, 2.0);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms;
            cudaEventElapsedTime(&ms, e0, e1);
            double fma = (double)sms * warps * iters * 16 * 32.0;
            if (rep) printf("DFMA warps/SM %2d: %.3f ms  %.2f TFLOP/s  (%.1f FMA/ns/SM)\n", warps, ms, 2 * fma / ms / 1e9, fma / ms / 1e6 / sms);
        }
    }
    // sustained: ~3 s of DMMA to see the power-capped clock
    cudaEventRecord(e0);
    for (int i = 0; i < 40; ++i) dmma_kernel<16><<<sms, 8 * 32>>>(out, iters * 4, 1.0, 2.0);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    double fma = 40.0 * sms * 8 * iters * 4 * 16 * 256.0;
    printf("DMMA sustained (%.0f ms): %.2f TFLOP/s\n", ms, 2 * fma / ms / 1e9);
    // the same for m16n8k4, the shape the GEMM kernels issue (~3 s at 66 TFLOP/s): the ceiling on a power-capped card
    cudaEventRecord(e0);
    for (int i = 0; i < 60; ++i) dmma16_kernel<8, 4><<<sms, 8 * 32>>>(out, iters * 16, 1.0, 2.0);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    fma = 60.0 * sms * 8 * iters * 16 * 8 * 512.0;
    printf("DMMA m16n8k4 sustained (%.0f ms): %.2f TFLOP/s\n", ms, 2 * fma / ms / 1e9);
    return 0;
}
