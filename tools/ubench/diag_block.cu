// Micro-benchmark: where the time of one 48x48 diagonal block of the team path goes (one CTA of 256 threads,
// shared memory, clock64 stamps).  Uses the production device functions.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I../../include -I../../aprilsam_b200/csrc -o diag_block diag_block.cu
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
struct BatchItem { unsigned long long dst; unsigned int off, bytes, fill, val; }; // as in asam_cuda.cu (k_step's item table)
#define ASAM_MAX_ITEMS 1024
#define ASAM_TABLE_BYTES (ASAM_MAX_ITEMS * sizeof(BatchItem))
#define ASAM_ITEM_CHUNK (8u << 10)
#include "asam_kernels.cuh"

__device__ __forceinline__ double rsqrt1(const double a)
{ // one Newton step from the float seed: ~2^-44 relative
    double y = (double) rsqrtf((float) a);
    double e = fma(-a * y, y, 1.0);
    return fma(0.5 * y, e, y);
}

// variant: same structure as panel_factor but with the one-step reciprocal square root
template <int NR>
__device__ __forceinline__ void pf_variant(double *P, int ldp, int k0, int pb, int m, double *dinv_out, int nt)
{
    const int tid = threadIdx.x;
    for (int c0 = 0; c0 < pb; c0 += 3) {
        const int rb = k0 + c0;
        double *p0 = P + (size_t) c0 * ldp, *p1 = p0 + ldp, *p2 = p1 + ldp;
        bar_sub(nt);
        const double a00 = p0[rb], a10 = p0[rb + 1], a20 = p0[rb + 2];
        const double a11 = p1[rb + 1], a21 = p1[rb + 2], a22 = p2[rb + 2];
        const double r0 = NR == 1 ? rsqrt1(a00) : d_rsqrt(a00);
        const double l10 = a10 * r0, l20 = a20 * r0;
        const double d1 = a11 - l10 * l10;
        const double r1 = NR == 1 ? rsqrt1(d1) : d_rsqrt(d1);
        const double l21 = (a21 - l20 * l10) * r1;
        const double d2 = a22 - l20 * l20 - l21 * l21;
        const double r2 = NR == 1 ? rsqrt1(d2) : d_rsqrt(d2);
        const int i_first = rb + 3 + tid;
        for (int i = i_first; i <= m; i += nt) {
            const double x0 = p0[i] * r0;
            const double x1 = (p1[i] - x0 * l10) * r1;
            const double x2 = (p2[i] - x0 * l20 - x1 * l21) * r2;
            p0[i] = x0; p1[i] = x1; p2[i] = x2;
        }
        bar_sub(nt);
        if (tid == 0) {
            p0[rb] = a00 * r0; p0[rb + 1] = l10; p0[rb + 2] = l20;
            p1[rb + 1] = d1 * r1; p1[rb + 2] = l21;
            p2[rb + 2] = d2 * r2;
            dinv_out[rb] = r0; dinv_out[rb + 1] = r1; dinv_out[rb + 2] = r2;
        }
        const int nrem = pb - (c0 + 3), nrow = m - (rb + 3) + 1;
        if (nrem > 0 && nrow > 0) {
            int ng = nt / nrow;
            ng = ng > nrem ? nrem : ng;
            const int gi = tid / nrow, ri = tid - gi * nrow;
            if (gi < ng) {
                const int i = rb + 3 + ri;
                const double x0 = p0[i], x1 = p1[i], x2 = p2[i];
                const int jmax = min(nrem, ri + 1);
                for (int jj = gi; jj < jmax; jj += ng) {
                    const int jr = rb + 3 + jj;
                    double *pj = P + (size_t) (c0 + 3 + jj) * ldp;
                    pj[i] -= x0 * p0[jr] + x1 * p1[jr] + x2 * p2[jr];
                }
            }
        }
    }
    bar_sub(nt);
}

__global__ void __launch_bounds__(256, 1) k_bench(const double *A, double *out, long long *st, int variant)
{
    __shared__ double D[48 * 48];
    __shared__ double rdv[48];
    __shared__ int err;
    const int tid = threadIdx.x;
    constexpr int LDD = 48;
    long long t[12];
    for (int rep = 0; rep < 3; rep++) {
        for (int e = tid; e < 48 * 48; e += 256)
            D[e] = A[e];
        if (tid == 0) err = 0;
        __syncthreads();
        t[0] = clock64();
        if (variant == 0) {
            diag_factor_rl(D, 48, rdv, 0, &err);
        } else if (variant == 1 || variant == 2) {
            for (int k1 = 0; k1 < 48; k1 += 12) {
                if (variant == 1) pf_variant<2>(D + (size_t) k1 * LDD, LDD, k1, 12, 47, rdv, 256);
                else pf_variant<1>(D + (size_t) k1 * LDD, LDD, k1, 12, 47, rdv, 256);
                if (k1 + 12 < 48) {
                    trailing_update<1, 4>(D, LDD, D + (size_t) k1 * LDD, LDD, 12, k1 + 12, 48, 47, 8);
                    bar_sub(256);
                }
            }
            __syncthreads();
        } else if (variant == 3) { // pieces
            t[1] = clock64();
            panel_factor(D, LDD, 0, 12, 47, 0, &err, rdv, 256);
            t[2] = clock64();
            trailing_update<1, 4>(D, LDD, D, LDD, 12, 12, 48, 47, 8);
            bar_sub(256);
            t[3] = clock64();
            for (int q = 0; q < 100; q++) bar_sub(256);
            t[4] = clock64();
            double v = A[tid] + 2.0;
            for (int q = 0; q < 100; q++) v = d_rsqrt(v) + 1.5;
            t[5] = clock64();
            for (int q = 0; q < 100; q++) v = rsqrt1(v) + 1.5;
            t[6] = clock64();
            for (int q = 0; q < 100; q++) v = fma(v, 0.999, 0.25);
            t[7] = clock64();
            for (int q = 0; q < 100; q++) { D[(tid * 7 + q) % 2304] = v; v = D[(tid * 13 + q * 5) % 2304] + 1.0; }
            t[8] = clock64();
            if (v == 12345.678) D[0] = v;
            __syncthreads();
        }
        t[9] = clock64();
    }
    if (tid == 0) {
        for (int q = 0; q < 10; q++) st[q] = t[q];
    }
    for (int e = tid; e < 48 * 48; e += 256)
        out[e] = D[e];
}

int main()
{
    const int n = 48;
    std::vector<double> A(n * n), B(n * n);
    srand(1);
    for (auto &v : B) v = rand() / (double) RAND_MAX - 0.5;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            double s = i == j ? 10.0 : 0.0;
            for (int k = 0; k < n; k++) s += B[i + k * n] * B[j + k * n];
            A[i + j * n] = s;
        }
    double *dA, *dO; long long *dS;
    cudaMalloc(&dA, sizeof(double) * n * n); cudaMalloc(&dO, sizeof(double) * n * n); cudaMalloc(&dS, 8 * 16);
    cudaMemcpy(dA, A.data(), sizeof(double) * n * n, cudaMemcpyHostToDevice);
    int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    std::vector<double> ref(n * n);
    for (int variant = 0; variant < 4; variant++) {
        // 0: production code (diag_factor_rl), the reference of the comparison; 1-3: variants / pieces
        k_bench<<<1, 256>>>(dA, dO, dS, variant);
        cudaError_t e = cudaDeviceSynchronize();
        long long st[10]; std::vector<double> O(n * n);
        cudaMemcpy(st, dS, sizeof(st), cudaMemcpyDeviceToHost);
        cudaMemcpy(O.data(), dO, sizeof(double) * n * n, cudaMemcpyDeviceToHost);
        if (variant == 0) ref = O;
        double md = 0;
        for (int j = 0; j < n; j++) for (int i = j; i < n; i++) md = fmax(md, fabs(O[i + j * n] - ref[i + j * n]) / fabs(ref[i + j * n]));
        printf("variant %d: %s  block %lld cycles (%.2f us at %d MHz)  max rel diff vs v0 %.2e\n", variant, cudaGetErrorString(e),
               st[9] - st[0], (st[9] - st[0]) / (khz * 1e-3), khz / 1000, md);
        if (variant == 3)
            printf("  pieces (cycles): panel_factor(12 cols, 48 rows) %lld, trailing 36x36 + bar %lld, bar_sub(256) %.1f, d_rsqrt+add %.1f, "
                   "rsqrt1+add %.1f, dependent DFMA %.1f, smem st+ld round trip %.1f\n",
                   st[2] - st[1], st[3] - st[2], (st[4] - st[3]) / 100.0, (st[5] - st[4]) / 100.0, (st[6] - st[5]) / 100.0,
                   (st[7] - st[6]) / 100.0, (st[8] - st[7]) / 100.0);
    }
    return 0;
}
