// Shared-memory wavefront probe: warp-wide LDS.32 / LDS.64 / LDS.128 with the address of lane l given by a pattern of
// its lane bits (the patterns the blend kernels use or could use).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lds_probe tools/lds_probe.cu
//   ncu --metrics l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum,smsp__inst_executed_op_shared_ld.sum \
//       --csv --log-file out.csv ./lds_probe 16 quick
// The wavefront counters of ncu are the measurement; the cycles the program prints itself are issue-bound (3 instructions
// per load) and only rank the patterns.  One CTA of NW warps per SM; every warp issues 8 independent loads per iteration.
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

template <int WIDTH>  // bytes per lane: 4, 8, 16
__global__ void probe(const int* __restrict__ lane_off, int iters, long long* cycles, float* sink) {
    extern __shared__ __align__(16) float sm[];
    for (int i = threadIdx.x; i < 8192; i += blockDim.x) sm[i] = (float)i;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // two 16 KB windows; every pattern stays below 12 KB
    uint32_t base = (uint32_t)__cvta_generic_to_shared(sm) + (warp & 1) * 16384 + lane_off[lane];
    uint32_t acc = 0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const uint32_t a = (base + u * 256) ^ ((it & 1) << 11);
            if (WIDTH == 16) {
                uint32_t x, y, z, w;
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a));
                acc += x + y;
                acc += z + w;
            } else if (WIDTH == 8) {
                uint32_t x, y;
                asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(x), "=r"(y) : "r"(a));
                acc += x + y;
            } else {
                uint32_t x;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(a));
                acc += x;
            }
        }
    }
    __syncthreads();
    const long long t1 = clock64();
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
    sink[blockIdx.x * blockDim.x + threadIdx.x] = (float)acc;
}

struct Pat { const char* name; int width; int (*f)(int); };
static int p_distinct16(int l) { return l * 16; }
static int p_and7_16(int l) { return (l & 7) * 16; }
static int p_shr3_16(int l) { return (l >> 3) * 16; }
static int p_and3_16(int l) { return (l & 3) * 16; }
static int p_same(int) { return 0; }
static int p_and15_16(int l) { return (l & 15) * 16; }
static int p_shr2_16(int l) { return (l >> 2) * 16; }
static int p_shr1_16(int l) { return (l >> 1) * 16; }
static int p_rows144(int l) { return (l & 7) * 144; }                 // 8 rows of a [entry][16 ch + 4 pad] slab
static int p_rows80_e8(int l) { return (l & 7) * 80; }                // rows of 20 floats, consecutive entries
static int p_rows144_q(int l) { return (l & 7) * 144 + (l >> 3) * 16; }  // 8 rows x 4 chunks: all distinct
static int p_distinct8(int l) { return l * 8; }
static int p_and15_8(int l) { return (l & 15) * 8; }
static int p_and7_8(int l) { return (l & 7) * 8; }
static int p_shr2_8(int l) { return (l >> 2) * 8; }
static int p_shr3_8(int l) { return (l >> 3) * 8; }
static int p_distinct4(int l) { return l * 4; }
static int p_and7_4(int l) { return (l & 7) * 4; }
static int p_shr3_4(int l) { return (l >> 3) * 4; }
static int p_stride8_4(int l) { return l * 32; }                       // 8-way... 32 B stride: 4-way bank conflict
static int p_and3_hi(int l) { return ((l & 3) | ((l >> 4) << 2)) * 16; }       // bits {4,1,0}: 8 chunks
static int p_b32(int l) { return (((l >> 2) & 3)) * 16; }                     // bits {3,2}: 4 chunks x 4 adjacent lanes, halves equal
static int p_b432(int l) { return (l >> 2) * 16; }                            // = lane>>2
static int p_b10_rows(int l) { return (l & 3) * 16 + ((l >> 4) & 1) * 64; }   // bits {4,1,0}
static int p_b1(int l) { return ((l >> 1) & 3) * 16; }                        // bits {2,1}: pairs adjacent, 4 chunks per quarter, quarters equal
static int p_b21_4(int l) { return (((l >> 1) & 3) | ((l >> 4) << 2)) * 16; } // bits {4,2,1}: 8 chunks
static int p_b0_3(int l) { return ((l & 1) | (((l >> 3) & 3) << 1)) * 16; }   // bits {4,3,0}: 8 chunks, 2 per quarter
static int p_b20(int l) { return (l & 1) * 16 + ((l >> 2) & 1) * 32; }        // bits {2,0}
static int g8(int l) { return (l & 1) | (((l >> 2) & 3) << 1); }
static int g4(int l) { return ((l >> 1) & 1) | ((l >> 4) << 1); }
static int p_g8_contig(int l) { return g8(l) * 16; }
static int p_g4_32(int l) { return g4(l) * 32; }
static int p_g8_1040(int l) { return g8(l) * 1040; }
static int p_g8_144(int l) { return g8(l) * 144; }
static int p_g4_144(int l) { return g4(l) * 144; }
static int p_g8_272(int l) { return g8(l) * 272; }
static int p_pairs16(int l) { return ((l & 7) * 2 + ((l >> 3) & 1)) * 16; }  // 16 distinct chunks, quarters 0/2 and 1/3 equal

int main(int argc, char** argv) {
    Pat pats[] = {
        {"v4 all distinct (512 B)", 16, p_distinct16}, {"v4 lane&7 (8 chunks, quarters equal)", 16, p_and7_16},
        {"v4 lane>>3 (4 chunks, one per quarter)", 16, p_shr3_16}, {"v4 lane&3 (4 chunks)", 16, p_and3_16},
        {"v4 all same", 16, p_same}, {"v4 lane&15 (16 chunks, halves equal)", 16, p_and15_16},
        {"v4 lane>>2 (8 chunks x4 lanes)", 16, p_shr2_16}, {"v4 lane>>1 (16 chunks x2 lanes)", 16, p_shr1_16},
        {"v4 8 rows stride 144 B, quarters equal", 16, p_rows144}, {"v4 8 rows stride 80 B, quarters equal", 16, p_rows80_e8},
        {"v4 8 rows stride 144 B x 4 chunks distinct", 16, p_rows144_q}, {"v4 16 chunks, quarter pairs equal", 16, p_pairs16},
        {"v4 bits{4,1,0}", 16, p_and3_hi}, {"v4 bits{3,2}", 16, p_b32}, {"v4 bits{2,1}", 16, p_b1},
        {"v4 bits{4,2,1}", 16, p_b21_4}, {"v4 bits{4,3,0}", 16, p_b0_3}, {"v4 bits{2,0}", 16, p_b20},
        {"v4 group8 contiguous (chain F)", 16, p_g8_contig}, {"v4 group4 x 32 B (chain D)", 16, p_g4_32},
        {"v4 group8 rows stride 1040 B (dfeature d)", 16, p_g8_1040}, {"v4 group8 rows stride 144 B", 16, p_g8_144},
        {"v4 group4 rows stride 144 B (dfeature w)", 16, p_g4_144}, {"v4 group8 rows stride 272 B", 16, p_g8_272},
        {"v2 all distinct (256 B)", 8, p_distinct8}, {"v2 lane&15", 8, p_and15_8}, {"v2 lane&7", 8, p_and7_8},
        {"v2 lane>>2", 8, p_shr2_8}, {"v2 lane>>3", 8, p_shr3_8},
        {"b32 all distinct", 4, p_distinct4}, {"b32 lane&7", 4, p_and7_4}, {"b32 lane>>3", 4, p_shr3_4},
        {"b32 stride 32 B (4-way conflict)", 4, p_stride8_4},
    };
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int* d_off; long long* d_cyc; float* d_sink;
    cudaMalloc(&d_off, 32 * 4); cudaMalloc(&d_cyc, sms * 8); cudaMalloc(&d_sink, sms * 1024 * 4);
    const int iters = argc > 1 ? atoi(argv[1]) : 4096;
    const bool quick = argc > 2;  // under ncu: one launch per pattern, 8 warps only
    cudaFuncSetAttribute(probe<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
    cudaFuncSetAttribute(probe<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
    cudaFuncSetAttribute(probe<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
    for (int nw : {8, 16}) {
        if (quick && nw != 8) break;
        printf("---- %d warps per SM\n", nw);
        for (auto& p : pats) {
            int off[32];
            for (int l = 0; l < 32; l++) off[l] = p.f(l);
            cudaMemcpy(d_off, off, sizeof(off), cudaMemcpyHostToDevice);
            for (int rep = 0; rep < (quick ? 1 : 2); rep++) {
                if (p.width == 16) probe<16><<<sms, nw * 32, 32768>>>(d_off, iters, d_cyc, d_sink);
                else if (p.width == 8) probe<8><<<sms, nw * 32, 32768>>>(d_off, iters, d_cyc, d_sink);
                else probe<4><<<sms, nw * 32, 32768>>>(d_off, iters, d_cyc, d_sink);
            }
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
            long long c; cudaMemcpy(&c, d_cyc, 8, cudaMemcpyDeviceToHost);
            printf("%-48s %6.2f cycles / warp-instruction\n", p.name, (double)c / ((double)iters * 8 * nw));
        }
    }
    return 0;
}
