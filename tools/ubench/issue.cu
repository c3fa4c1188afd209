// Issue-rate microbenchmarks for the mixing walker's design: what ONE warp can issue per cycle, per pipe and across
// pipes (lat.cu measures dependent-chain latencies; this measures streams of independent instructions).  Every case
// runs 8 independent register chains (chain k reads chain k+1's value of the previous step, >= 7 instructions old), so
// latency does not bound it; the result is cycles per instruction of the stream.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o issue issue.cu ; run on an H100.
// tools/ubench/issue_sass.py prints the opcode histogram of every case's loop body (the intended opcode and the loop's
// own counter/branch must be all there is).
// Two block shapes: 32 threads (a lone warp) and 128 threads of which warps 1..3 exit after the first barrier, as the
// helper warps of the walker (W2_THREADS = 128) do after its prologue.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define ITER 512
#define ROUNDS 4   // steps of all 8 chains per loop iteration
__device__ __forceinline__ long long clk() { long long c; asm volatile("mov.u64 %0, %%clock64;" : "=l"(c)); return c; }

enum Case {
    C_LOP3, C_SHF, C_IADD3, C_ISETP_SEL, C_PRMT, C_FSETP_FSEL, C_FMNMX,           // ALU pipe
    C_FADD, C_FFMA, C_FMUL, C_IMAD, C_IMAD_IADD, C_IMAD_SHLADD,                   // FMA pipe (the last two: forms the compiler picks itself)
    C_ULOP3, C_USHF, C_UIADD3, C_UPOPC, C_VOTE, C_VOTEU,                          // uniform datapath
    C_LDS32, C_LDS64, C_LDS64_PERM, C_LDS_U16, C_LDS_U8, C_STS64, C_CP_ASYNC,     // LSU
    C_STS64_8L,                                                                   // 8 of 32 lanes active, as in the walker's commit
    C_POPC, C_SHFL,
    C_MIX_ALU_FMA, C_MIX_ALU_IMAD, C_MIX_FFMA_IMAD, C_MIX_ALU_UNI, C_MIX_ALU_LDS, C_MIX_FMA_UNI, C_MIX_ALU_FMA_UNI,
    C_COUNT
};

template <class F>
__device__ __forceinline__ void stream8(unsigned (&x)[8], F f) {
#pragma unroll 1
    for (int n = 0; n < ITER; n++) {
#pragma unroll
        for (int r = 0; r < ROUNDS; r++) {
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = f(x[k], x[(k + 1) & 7]);
        }
    }
}
// two streams, interleaved 1:1
template <class F, class G>
__device__ __forceinline__ void stream8x2(unsigned (&x)[8], unsigned (&y)[8], F f, G g) {
#pragma unroll 1
    for (int n = 0; n < ITER; n++) {
#pragma unroll
        for (int r = 0; r < ROUNDS; r++) {
#pragma unroll
            for (int k = 0; k < 8; k++) { x[k] = f(x[k], x[(k + 1) & 7]); y[k] = g(y[k], y[(k + 1) & 7]); }
        }
    }
}
template <class F, class G, class H>
__device__ __forceinline__ void stream8x3(unsigned (&x)[8], unsigned (&y)[8], unsigned (&z)[8], F f, G g, H h) {
#pragma unroll 1
    for (int n = 0; n < ITER; n++) {
#pragma unroll
        for (int r = 0; r < ROUNDS; r++) {
#pragma unroll
            for (int k = 0; k < 8; k++) {
                x[k] = f(x[k], x[(k + 1) & 7]); y[k] = g(y[k], y[(k + 1) & 7]); z[k] = h(z[k], z[(k + 1) & 7]);
            }
        }
    }
}

#define FU(v) __uint_as_float(v)
#define UF(v) __float_as_uint(v)

template <int C>
__global__ void k_issue(unsigned seed, long long *out, unsigned *sink, const uint4 *gsrc) {
    __shared__ __align__(16) unsigned sm[2048];
    const int lane = threadIdx.x & 31;
    for (int q = threadIdx.x; q < 2048; q += blockDim.x) sm[q] = q * 97u + seed;
    __syncthreads();
    if (threadIdx.x >= 32) return;   // the helper warps are gone from here on
    const unsigned sbase = (unsigned)__cvta_generic_to_shared((const void *)sm);
    unsigned x[8], y[8], z[8];
    for (int k = 0; k < 8; k++) {
        x[k] = seed * (2 * k + 3) + lane * 0x9e3779b9u;                                       // per lane
        y[k] = UF(1.0f + 0.001f * (float)((seed + k + lane) & 63));                           // per lane, float bits
        z[k] = __ballot_sync(0xffffffffu, ((seed * (k + 5)) >> lane) & 1u) ^ (seed << k);     // warp-uniform
    }
    const unsigned c = seed ^ (lane * 0x85ebca6bu), cu = seed * 0x27d4eb2fu;
    const float cf = 1.0f + 1e-7f * (float)lane;
    // ALU-pipe, FMA-pipe and uniform-datapath steps (uniform: all inputs are warp-wide values, so the compiler may place
    // the chain on the uniform datapath; issue_sass.py shows whether it did)
    auto lop3 = [&](unsigned a, unsigned b) { unsigned d; asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; };
    auto ffma = [&](unsigned a, unsigned b) { return UF(fmaf(FU(a), cf, FU(b))); };
    auto imad = [&](unsigned a, unsigned b) { unsigned d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(c), "r"(b)); return d; };
    auto ulop3 = [&](unsigned a, unsigned b) { return (a ^ b) | cu; };
    long long t0 = 0, t1 = 0;
    int ops = 8 * ROUNDS;   // instructions of interest per loop iteration
    t0 = clk();
    if constexpr (C == C_LOP3) stream8(x, lop3);
    else if constexpr (C == C_SHF) stream8(x, [&](unsigned a, unsigned b) { return __funnelshift_r(a, b, c); });
    else if constexpr (C == C_IADD3) stream8(x, [&](unsigned a, unsigned b) { return a + b + c; });
    else if constexpr (C == C_ISETP_SEL) { stream8(x, [&](unsigned a, unsigned b) { return a > b ? a ^ 0u : c; }); ops *= 2; }
    else if constexpr (C == C_PRMT) stream8(x, [&](unsigned a, unsigned b) { return __byte_perm(a, b, 0x1045); });
    else if constexpr (C == C_FSETP_FSEL) { stream8(y, [&](unsigned a, unsigned b) { return FU(a) > FU(b) ? a : UF(cf); }); ops *= 2; }
    else if constexpr (C == C_FMNMX) stream8(y, [&](unsigned a, unsigned b) { return UF(fminf(FU(a), FU(b))); });
    else if constexpr (C == C_FADD) stream8(y, [&](unsigned a, unsigned b) { return UF(FU(a) + FU(b)); });
    else if constexpr (C == C_FFMA) stream8(y, ffma);
    else if constexpr (C == C_FMUL) stream8(y, [&](unsigned a, unsigned b) { return UF(FU(a) * FU(b)); });
    else if constexpr (C == C_IMAD) stream8(x, imad);
    else if constexpr (C == C_IMAD_IADD) stream8(x, [&](unsigned a, unsigned b) { return a + b; });
    else if constexpr (C == C_IMAD_SHLADD) stream8(x, [&](unsigned a, unsigned b) { return (a << 3) + b; });
    else if constexpr (C == C_ULOP3) stream8(z, ulop3);
    else if constexpr (C == C_USHF) stream8(z, [&](unsigned a, unsigned b) { return __funnelshift_r(a, b, cu); });
    else if constexpr (C == C_UIADD3) stream8(z, [&](unsigned a, unsigned b) { return a + b; });
    else if constexpr (C == C_UPOPC) stream8(z, [&](unsigned a, unsigned b) { return (unsigned)__popc(b); });
    else if constexpr (C == C_VOTE) {   // per-lane test of the neighbour chain's word, ballot into a vector register
        stream8(x, [&](unsigned a, unsigned b) { return __ballot_sync(0xffffffffu, (b & c) != 0u); });
        ops *= 2;   // LOP3 (to a predicate) + VOTE
    } else if constexpr (C == C_VOTEU) {   // the same with a warp-wide word and the walker's rotation of the ballot
        stream8(z, [&](unsigned a, unsigned b) { const unsigned v = __ballot_sync(0xffffffffu, (b & c) != 0u); return __funnelshift_r(v, v, cu); });
        ops *= 3;   // LOP3 (to a predicate) + VOTE + SHF: the compiler keeps this ballot in a vector register
    } else if constexpr (C == C_LDS32 || C == C_LDS64 || C == C_LDS64_PERM || C == C_LDS_U16 || C == C_LDS_U8) {
        const unsigned a = sbase + (C == C_LDS32 ? lane * 4 : C == C_LDS64 ? lane * 8 : C == C_LDS64_PERM ? ((lane * 37 + seed) & 255) * 8
                                    : C == C_LDS_U16 ? lane * 2 : lane);
#pragma unroll 1
        for (int n = 0; n < ITER; n++) {
#pragma unroll
            for (int k = 0; k < 8 * ROUNDS; k++) {
                if constexpr (C == C_LDS32) asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(x[k & 7]) : "r"(a));
                else if constexpr (C == C_LDS_U16) asm volatile("ld.volatile.shared.u16 %0, [%1];" : "=r"(x[k & 7]) : "r"(a));
                else if constexpr (C == C_LDS_U8) asm volatile("ld.volatile.shared.u8 %0, [%1];" : "=r"(x[k & 7]) : "r"(a));
                else asm volatile("ld.volatile.shared.v2.u32 {%0, %1}, [%2];" : "=r"(x[k & 7]), "=r"(y[k & 7]) : "r"(a));
            }
        }
    } else if constexpr (C == C_STS64) {
        const unsigned a = sbase + lane * 8;
#pragma unroll 1
        for (int n = 0; n < ITER; n++) {
#pragma unroll
            for (int k = 0; k < 8 * ROUNDS; k++) asm volatile("st.volatile.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x[k & 7]), "r"(y[k & 7]) : "memory");
        }
    } else if constexpr (C == C_STS64_8L) {
        const unsigned a = sbase + lane * 8;
#pragma unroll 1
        for (int n = 0; n < ITER; n++) {
#pragma unroll
            for (int k = 0; k < 8 * ROUNDS; k++)
                asm volatile("{ .reg .pred p; setp.lt.u32 p, %3, 8; @p st.volatile.shared.v2.u32 [%0], {%1, %2}; }" ::"r"(a), "r"(x[k & 7]), "r"(y[k & 7]), "r"(lane) : "memory");
        }
    } else if constexpr (C == C_CP_ASYNC) {   // 16-byte copies, one group per 8, at most 2 groups in flight
        const unsigned a = sbase + lane * 16;
#pragma unroll 1
        for (int n = 0; n < ITER; n++) {
#pragma unroll
            for (int r = 0; r < ROUNDS; r++) {
#pragma unroll
                for (int k = 0; k < 8; k++) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(a + 512 * (k & 3)), "l"(gsrc + lane + 32 * k) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 2;" ::: "memory");
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    } else if constexpr (C == C_POPC) stream8(x, [&](unsigned a, unsigned b) { return (unsigned)__popc(b); });
    else if constexpr (C == C_SHFL) stream8(x, [&](unsigned a, unsigned b) { return __shfl_xor_sync(0xffffffffu, b, 1); });
    else if constexpr (C == C_MIX_ALU_FMA) { stream8x2(x, y, lop3, ffma); ops *= 2; }
    else if constexpr (C == C_MIX_ALU_IMAD) { unsigned v[8]; for (int k = 0; k < 8; k++) v[k] = x[k] * 3u + 1u; stream8x2(x, v, lop3, imad); for (int k = 0; k < 8; k++) y[k] ^= v[k]; ops *= 2; }
    else if constexpr (C == C_MIX_FFMA_IMAD) { stream8x2(y, x, ffma, imad); ops *= 2; }
    else if constexpr (C == C_MIX_ALU_UNI) { stream8x2(x, z, lop3, ulop3); ops *= 2; }
    else if constexpr (C == C_MIX_ALU_LDS) {
        const unsigned a = sbase + lane * 4;
        unsigned v = 0;
#pragma unroll 1
        for (int n = 0; n < ITER; n++) {
#pragma unroll
            for (int r = 0; r < ROUNDS; r++) {
#pragma unroll
                for (int k = 0; k < 8; k++) { x[k] = lop3(x[k], x[(k + 1) & 7]); asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); }
            }
        }
        y[0] ^= v;
        ops *= 2;
    } else if constexpr (C == C_MIX_FMA_UNI) { stream8x2(y, z, ffma, ulop3); ops *= 2; }
    else if constexpr (C == C_MIX_ALU_FMA_UNI) { stream8x3(x, y, z, lop3, ffma, ulop3); ops *= 3; }
    t1 = clk();
    unsigned acc = 0;
    for (int k = 0; k < 8; k++) acc ^= x[k] ^ y[k] ^ z[k];
    sink[threadIdx.x] = acc;
    if (lane == 0) { out[2 * C] = t1 - t0; out[2 * C + 1] = (long long)ops * ITER; }
}

static const char *names[C_COUNT] = {
    "LOP3", "SHF", "IADD3", "ISETP+SEL (per instruction)", "PRMT", "FSETP+FSEL (per instruction)", "FMNMX",
    "FADD", "FFMA", "FMUL", "IMAD", "two-input add (IMAD.IADD 7 : IADD3 1)", "shift-add (IMAD 7 : LEA 1)",
    "ULOP3", "USHF", "UIADD3", "UPOPC", "LOP3+VOTE (per instruction)", "LOP3+VOTE+SHF rotate (per instruction)",
    "LDS.32", "LDS.64", "LDS.64 permuted 8-byte stride", "LDS.U16", "LDS.U8", "STS.64", "cp.async 16 B (LDGSTS)", "STS.64, 8 lanes active",
    "POPC", "SHFL",
    "mix LOP3 : FFMA", "mix LOP3 : IMAD", "mix FFMA : IMAD", "mix LOP3 : ULOP3", "mix LOP3 : LDS.32", "mix FFMA : ULOP3", "mix LOP3 : FFMA : ULOP3"};

template <int C>
static void run_all(int threads, long long *out, unsigned *sink, const uint4 *gsrc) {
    if constexpr (C < C_COUNT) {
        k_issue<C><<<1, threads>>>(12345u, out, sink, gsrc);
        run_all<C + 1>(threads, out, sink, gsrc);
    }
}

int main() {
    long long *out; unsigned *sink; uint4 *gsrc;
    cudaMallocManaged(&out, 2 * C_COUNT * sizeof(long long)); cudaMalloc(&sink, 1024 * 4); cudaMalloc(&gsrc, 4096 * 16);
    cudaMemset(gsrc, 1, 4096 * 16);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    printf("device: %s, %d SMs, %d MHz max SM clock (power limit: see nvidia-smi --query-gpu=power.limit)\n", p.name, p.multiProcessorCount, p.clockRate / 1000);
    const int shapes[2] = {32, 128};
    for (int m = 0; m < 2; m++) {
        printf("-- block of %d threads%s\n", shapes[m], m ? " (warps 1..3 exit after the first barrier)" : " (a lone warp)");
        for (int rep = 0; rep < 2; rep++) {
            run_all<0>(shapes[m], out, sink, gsrc);
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { printf("error: %s\n", cudaGetErrorString(e)); return 1; }
        }
        for (int c = 0; c < C_COUNT; c++) printf("%-42s %6.2f cycles/instruction\n", names[c], (double)out[2 * c] / (double)out[2 * c + 1]);
    }
    return 0;
}
