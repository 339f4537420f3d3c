// libfcma_b200.so — Hopper-native (sm_90a) FCMA correlation engine behind a C ABI.
//
// Path (reference brainiak/brainiak @ 123f6e1):
//   a14  preprocessing.py:80-84      per-epoch z-score                -> k_pack_operand (normalise prologue)
//   a4   voxelselector.py:307-323    E skinny SGEMMs                  -> k_corr_wgmma  (TMA + wgmma)
//   a6   fcma_extension.cc:52-84     Fisher-z + within-subject zscore -> k_norm_syrk   (fused with a7)
//   a7   voxelselector.py:400-408    per-voxel SSYRK                  -> k_norm_syrk   (mma.sync tf32)
//   a9-a11 classifier.py:279-348     same, one [E,E] kernel           -> k_norm_syrk + k_reduce_rows
// plus standalone, reference-exact stages (k_within_subject_norm, k_corr_simt, k_syrk_simt).
//
// No CPU fallback lives here: without an sm_90 device every compute entry point returns FCMA_ENODEV.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>

#include <atomic>
#include <mutex>

#include "../../include/fcma_b200.h"
#include "ptx_sm90.cuh"

using namespace fcma;

// ============================================================================================
// host-side helpers
// ============================================================================================
static thread_local char g_err[512] = "";
static std::atomic<long> g_launches{0};

static int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_TRY(expr)                                                                           \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess)                                                                   \
            return fail(FCMA_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                        __LINE__);                                                               \
    } while (0)
#define LAUNCH_CHECK(name)                                                                       \
    do {                                                                                         \
        g_launches.fetch_add(1, std::memory_order_relaxed);                                      \
        cudaError_t _e = cudaGetLastError();                                                     \
        if (_e != cudaSuccess)                                                                   \
            return fail(FCMA_ECUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e));    \
    } while (0)

static inline long cdiv(long a, long b) { return (a + b - 1) / b; }
static inline long round_up(long a, long b) { return cdiv(a, b) * b; }

// Launches kernel<<<grid, block, smem, st>>>(args...) and counts it; a kernel that needs more than the default 48 KB of
// dynamic shared memory gets its limit raised first.
template <typename... Params, typename... Args>
static int launch_kernel(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const char *name,
                         Args... args)
{
    if (smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, block, smem, st>>>(args...);
    LAUNCH_CHECK(name);
    return FCMA_OK;
}

// Calls f(IntC<V>{}) for the V of the list that equals `value`, so that a kernel template is instantiated for exactly the
// listed values.  Returns false when the list has no such V.
template <int V>
using IntC = std::integral_constant<int, V>;
template <int... Vs, typename F>
static bool with_int(int value, F &&f)
{
    return ((value == Vs && (f(IntC<Vs>{}), true)) || ...);
}

// Tuning / diagnostic knobs (A/B switches of tools/) exist only in the diagnostic build (-DFCMA_DIAG -> libfcma_b200_diag.so, `python -m brainiak_b200.build --diag`).  The
// product library never reads the environment: a stray variable cannot change its numerics or layout.
#ifdef FCMA_DIAG
static inline const char *diag_env(const char *name) { return getenv(name); }
#else
static inline const char *diag_env(const char *) { return nullptr; }
#endif

// RAII holders so that early error returns do not leak stream-ordered allocations or events
struct AsyncBuf {
    void *p = nullptr;
    cudaStream_t st = nullptr;
    ~AsyncBuf()
    {
        if (p) cudaFreeAsync(p, st);
    }
    cudaError_t alloc(size_t n, cudaStream_t s)
    {
        st = s;
        return cudaMallocAsync(&p, n ? n : 1, s);
    }
};
template <int N>
struct EventSet {
    cudaEvent_t ev[N] = {};
    bool on = false;
    ~EventSet()
    {
        for (int k = 0; k < N; k++)
            if (ev[k]) cudaEventDestroy(ev[k]);
    }
    cudaError_t create()
    {
        on = true;
        for (int k = 0; k < N; k++) {
            cudaError_t e = cudaEventCreate(&ev[k]);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
};
// restores the caller's current device when a host-buffer entry point returns (they run on `device`)
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; } }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int g_sm_count = 0;
static int check_device()
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(FCMA_ENODEV, "no CUDA device: %s", cudaGetErrorString(e));
    }
    static thread_local int checked_dev = -1;
    if (checked_dev == dev) return FCMA_OK;
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(FCMA_ENODEV, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    }
    if (prop.major != 9)
        return fail(FCMA_ENODEV, "device %d is sm_%d%d; libfcma_b200 needs sm_90 (H100)", dev, prop.major,
                    prop.minor);
    g_sm_count = prop.multiProcessorCount;
    checked_dev = dev;
    return FCMA_OK;
}

extern "C" int fcma_version(void) { return 100; }
extern "C" const char *fcma_last_error(void) { return g_err; }
extern "C" long fcma_launch_count(void) { return g_launches.load(); }
extern "C" int fcma_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int d = 0; d < n; d++) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess && major == 9)
            ok++;
    }
    return ok;
}

// ============================================================================================
// precision descriptors
// ============================================================================================
struct PrecInfo {
    int planes;    // stored planes (hi[, lo])
    int segs;      // product segments
    int seg_r[3];  // plane of the row operand per segment
    int seg_c[3];  // plane of the column operand per segment
    int esize;     // bytes per element
    int bk;        // K elements per 128-byte swizzle row (TMA box width)
    int mma_k;     // K per wgmma
    int fmt;       // operand type of the wgmma: 0 f16, 1 bf16, 2 tf32
    int pack;      // element type written by k_pack_operand: 0 bf16, 1 tf32-rounded fp32, 2 fp16 (scaled)
    float in_scale;  // operands are stored multiplied by this power of two (fp16 range management)
};
// fp16 planes hold x * 2^6: |x| <= 1 for normalised epochs, so hi <= 64 and the low plane
// (~2^-11 of hi) stays a NORMAL fp16 number down to |x| ~ 4e-3; the epilogue multiplies by 2^-12.
constexpr float FCMA_FP16_SCALE = 64.0f;
static bool prec_info(int precision, PrecInfo *p)
{
    switch (precision) {
    case FCMA_PREC_BF16: *p = {1, 1, {0, 0, 0}, {0, 0, 0}, 2, 64, 16, 1, 0, 1.0f}; return true;
    case FCMA_PREC_TF32: *p = {1, 1, {0, 0, 0}, {0, 0, 0}, 4, 32, 8, 2, 1, 1.0f}; return true;
    // small cross terms first, hi*hi last
    case FCMA_PREC_BF16X3: *p = {2, 3, {1, 0, 0}, {0, 1, 0}, 2, 64, 16, 1, 0, 1.0f}; return true;
    case FCMA_PREC_TF32X3: *p = {2, 3, {1, 0, 0}, {0, 1, 0}, 4, 32, 8, 2, 1, 1.0f}; return true;
    case FCMA_PREC_FP16X3: *p = {2, 3, {1, 0, 0}, {0, 1, 0}, 2, 64, 16, 0, 2, FCMA_FP16_SCALE}; return true;
    default: return false;
    }
}
extern "C" int fcma_operand_kp(int precision, int T)
{
    PrecInfo p;
    if (!prec_info(precision, &p) || T <= 0) return 0;
    return (int)round_up(T, p.mma_k);  // bf16: multiple of 16 (32 B); tf32: multiple of 8 (32 B)
}
extern "C" int fcma_operand_planes(int precision)
{
    PrecInfo p;
    return prec_info(precision, &p) ? p.planes : 0;
}
// bytes of the K-major planes, rounded up so that the trailing [E][V] fp32 self-correlation diagonal
// (exact sequential-FMA sum of squares, see k_pack_operand) stays 256-byte aligned
static size_t operand_plane_bytes(const PrecInfo &p, int precision, int E, int T, long V)
{
    size_t b = (size_t)p.planes * E * V * fcma_operand_kp(precision, T) * p.esize;
    return (b + 255) & ~(size_t)255;
}
extern "C" size_t fcma_operand_bytes(int precision, int E, int T, long V)
{
    PrecInfo p;
    if (!prec_info(precision, &p)) return 0;
    return operand_plane_bytes(p, precision, E, T, V) + (size_t)E * V * sizeof(float);
}

// ============================================================================================
// a14 + operand packing:  [E][T][ld] fp32 (voxels contiguous)  ->  [planes][E][V][Kp] K-major
// ============================================================================================
__device__ __forceinline__ float tf32_rn(float x)
{
    return __uint_as_float(f32_to_tf32(x));
}

// one block = 32 voxels of one epoch; 256 threads = 32 (voxel) x 8
template <int KIND, int PLANES>
__global__ void __launch_bounds__(256) k_pack_operand(const float *__restrict__ src, int E, int T, long V, long ld,
                                                      const int *__restrict__ T_e, int normalize, void *dst, int Kp,
                                                      float *__restrict__ selfdiag, float in_scale, long v_begin, long v_end, int e_begin)
{
    __shared__ double s_red[8][33];
    __shared__ float s_mean[32], s_scale[32];
    __shared__ float s_tile[32][65];
    const int e = e_begin + blockIdx.y;          // grid.y = epochs packed by this launch
    const long v0 = v_begin + (long)blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int Te = T_e ? T_e[e] : T;
    const float *ep = src + (size_t)e * T * ld;
    const long v = v0 + tx;
    const bool vok = v < v_end;   // voxels [v_begin, v_end) of the V-voxel layout

    float mean = 0.f, scale = 1.f;
    if (normalize) {
        // two-pass mean / population std over the Te rows (numpy semantics of zscore(ddof=0))
        double s = 0.0;
        for (int t = ty; t < Te; t += 8) s += vok ? (double)ep[(size_t)t * ld + v] : 0.0;
        s_red[ty][tx] = s;
        __syncthreads();
        if (ty == 0) {
            double tot = 0.0;
            for (int k = 0; k < 8; k++) tot += s_red[k][tx];
            s_mean[tx] = (float)(tot / Te);
        }
        __syncthreads();
        mean = s_mean[tx];
        double q = 0.0;
        for (int t = ty; t < Te; t += 8) {
            float d = vok ? ep[(size_t)t * ld + v] - mean : 0.f;
            q += (double)d * d;
        }
        __syncthreads();
        s_red[ty][tx] = q;
        __syncthreads();
        if (ty == 0) {
            double tot = 0.0;
            for (int k = 0; k < 8; k++) tot += s_red[k][tx];
            float sd = (float)sqrt(tot / Te);
            // (x-mean)/sd: sd == 0 -> 0/0 = nan -> nan_to_num -> 0; then / sqrt(Te)
            s_scale[tx] = sd > 0.f ? 1.0f / (sd * sqrtf((float)Te)) : 0.f;
        }
        __syncthreads();
        scale = s_scale[tx];
    }

    // Exact self-correlation of each voxel: the reference's sgemm (OpenBLAS FMA micro-kernel) is
    // bit-identical to a sequential fp32 FMA chain over t (verified against reference outputs,
    // tests/golden), so this reproduces its r[i,e,i] = 1 +- ulp rounding pattern exactly.  Warp 0 runs the chain
    // on the values of each slab while they sit in shared memory (rows t >= Te hold 0 and leave it unchanged):
    // no extra pass over the epoch in HBM.
    float diag_acc = 0.f;
    const size_t plane_stride = (size_t)E * V * Kp;
    for (int k0 = 0; k0 < Kp; k0 += 64) {
        // load a [64 t][32 v] slab coalesced along v, transpose through smem
        for (int tt = ty; tt < 64; tt += 8) {
            int t = k0 + tt;
            float x = 0.f;
            if (t < Te && vok) {
                x = ep[(size_t)t * ld + v];
                if (normalize) {
                    x = (x - mean) * scale;
                    if (!(x == x)) x = 0.f;  // nan_to_num (nan inputs)
                }
            }
            s_tile[tx][tt] = x;
        }
        __syncthreads();
        if (ty == 0) {
#pragma unroll 16
            for (int tt = 0; tt < 64; tt++) {
                const float x = s_tile[tx][tt];
                diag_acc = fmaf(x, x, diag_acc);
            }
        }
        // 8 warps x 4 voxels; a warp writes 64 consecutive k of one voxel row
        for (int vv = ty * 4; vv < ty * 4 + 4; vv++) {
            long vo = v0 + vv;
            if (vo >= v_end) continue;
            for (int kk = tx; kk < 64; kk += 32) {
                int k = k0 + kk;
                if (k >= Kp) continue;
                float x = s_tile[vv][kk];
                size_t off = ((size_t)e * V + vo) * Kp + k;
                if constexpr (KIND == 0) {
                    __nv_bfloat16 *d = reinterpret_cast<__nv_bfloat16 *>(dst);
                    __nv_bfloat16 hi = __float2bfloat16_rn(x);
                    d[off] = hi;
                    if constexpr (PLANES > 1) d[plane_stride + off] = __float2bfloat16_rn(x - __bfloat162float(hi));
                } else if constexpr (KIND == 2) {
                    __half *d = reinterpret_cast<__half *>(dst);
                    const float xs = x * in_scale;               // exact (power of two)
                    __half hi = __float2half_rn(xs);
                    d[off] = hi;
                    if constexpr (PLANES > 1) d[plane_stride + off] = __float2half_rn(xs - __half2float(hi));
                } else {
                    float *d = reinterpret_cast<float *>(dst);
                    float hi = tf32_rn(x);
                    d[off] = hi;
                    if constexpr (PLANES > 1) d[plane_stride + off] = tf32_rn(x - hi);
                }
            }
        }
        __syncthreads();
    }
    if (ty == 0 && vok) selfdiag[(size_t)e * V + v] = diag_acc;
}

// a14 in place on [E][T][ld]
__global__ void __launch_bounds__(256) k_epoch_normalize(float *data, int T, long V, long ld, const int *__restrict__ T_e)
{
    __shared__ double s_red[8][33];
    __shared__ float s_mean[32], s_scale[32];
    const int e = blockIdx.y;
    const long v = (long)blockIdx.x * 32 + (threadIdx.x & 31);
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int Te = T_e ? T_e[e] : T;
    float *ep = data + (size_t)e * T * ld;
    const bool vok = v < V;
    double s = 0.0;
    for (int t = ty; t < Te; t += 8) s += vok ? (double)ep[(size_t)t * ld + v] : 0.0;
    s_red[ty][tx] = s;
    __syncthreads();
    if (ty == 0) {
        double tot = 0.0;
        for (int k = 0; k < 8; k++) tot += s_red[k][tx];
        s_mean[tx] = (float)(tot / Te);
    }
    __syncthreads();
    float mean = s_mean[tx];
    double q = 0.0;
    for (int t = ty; t < Te; t += 8) {
        float d = vok ? ep[(size_t)t * ld + v] - mean : 0.f;
        q += (double)d * d;
    }
    __syncthreads();
    s_red[ty][tx] = q;
    __syncthreads();
    if (ty == 0) {
        double tot = 0.0;
        for (int k = 0; k < 8; k++) tot += s_red[k][tx];
        float sd = (float)sqrt(tot / Te);
        s_scale[tx] = sd > 0.f ? 1.0f / (sd * sqrtf((float)Te)) : 0.f;
    }
    __syncthreads();
    float scale = s_scale[tx];
    if (vok)
        for (int t = ty; t < Te; t += 8) {
            float x = (ep[(size_t)t * ld + v] - mean) * scale;
            if (!(x == x)) x = 0.f;
            ep[(size_t)t * ld + v] = x;
        }
}

// ============================================================================================
// a4 on tensor cores: persistent, warp-specialised TMA -> wgmma (accumulators in registers) -> HBM
// ============================================================================================

__device__ __forceinline__ float rsqrt_ftz(float x)
{
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float lg2_ftz(float x)
{
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// log2((1+r)/(1-r)) with the reference's clamps: Fisher-z up to the factor 0.5*ln2, which the
// within-subject z-score that follows cancels exactly
__device__ __forceinline__ float fisher_log2(float r)
{
    float num = 1.0f + r, den = 1.0f - r;
    num = num <= 0.f ? 1e-4f : num;
    den = den <= 0.f ? 1e-4f : den;
    return lg2_ftz(num) - lg2_ftz(den);
}
__device__ __forceinline__ float fisher_fast(float r)
{
    // 0.5*log((1+r)/(1-r)) with the clamps of fcma_extension.cc:68-72, as 0.5*ln2*(lg2(num)-lg2(den))
    float num = 1.0f + r, den = 1.0f - r;
    num = num <= 0.f ? 1e-4f : num;
    den = den <= 0.f ? 1e-4f : den;
    return 0.34657359027997264f * (lg2_ftz(num) - lg2_ftz(den));
}

// mean^2 - E[x^2] of a subject's EPS values from nm = -mean and ns2 = -E[x^2], as one FMA.  EPS == 1: exactly 0, as in
// fcma_extension.cc (x*x/1 - x*x); the FMA would return the rounding error of x^2, and its rsqrt z-scores of up to ~1
template <int EPS>
__device__ __forceinline__ float2 neg_variance(float2 nm, float2 ns2)
{
    if constexpr (EPS == 1)
        return splat2(0.f);
    else
        return ffma2(nm, nm, ns2);
}

// GEMM-epilogue Fisher-z, series form: atanh(r) = r + r^3/3 + ... + r^13/13 for |r| <= 0.35 (truncation
// < 3e-8 relative; 9 FMA-pipe ops, no MUFU).  The epilogue takes it for a whole warp block when no
// element exceeds the bound (warp vote; r ~ N(0, 1/sqrt(T)) makes that the common case) and the
// two-logarithm form with the reference's clamps otherwise: fisher_fast costs two XU ops per element.
constexpr float FISHER_SERIES_MAX = 0.35f;
// scalar form, bit-identical to one lane of fisher_series2 (same fma.rn sequence)
__device__ __forceinline__ float fisher_series1(float r)
{
    const float x2 = fmaf(r, r, 0.f);
    float p = fmaf(0.076923076923f, x2, 0.090909090909f);
    p = fmaf(p, x2, 0.111111111111f);
    p = fmaf(p, x2, 0.142857142857f);
    p = fmaf(p, x2, 0.2f);
    p = fmaf(p, x2, 0.333333333333f);
    return fmaf(fmaf(r, x2, 0.f), p, r);
}
// two accumulators at once (packed fp32x2 FMAs): returns atanh(a * scale)
__device__ __forceinline__ float2 fisher_series2(float2 a, float scale)
{
    const float2 zero = splat2(0.f);
    const float2 r = ffma2(a, splat2(scale), zero);
    const float2 x2 = ffma2(r, r, zero);
    float2 p = ffma2(splat2(0.076923076923f), x2, splat2(0.090909090909f));   // 1/13, 1/11
    p = ffma2(p, x2, splat2(0.111111111111f));                                 // 1/9
    p = ffma2(p, x2, splat2(0.142857142857f));                                 // 1/7
    p = ffma2(p, x2, splat2(0.2f));
    p = ffma2(p, x2, splat2(0.333333333333f));
    return ffma2(ffma2(r, x2, zero), p, r);
}

// ---------------------------------------------------------------- correlation tiles on wgmma
// One CTA computes 128 columns j (wgmma M side, two consumer warpgroups of 64) x 256 rows i (wgmma N side) of one
// epoch; two CTAs (blockIdx.x & 1 = `half`) cover a 256 x 256 tile.  The operands are K-major, 128-byte swizzled
// [voxel][Kp] tiles, exactly the boxes the packer's layout gives TMA.  In the 3-product modes one stage carries
// {cols_hi, cols_lo, rows_hi, rows_lo} of a k-block and feeds all three products.
//   warpgroup 0   : one elected thread issues the TMA loads into a ring of `stages` stages (full / empty mbarriers)
//   warpgroups 1-2: wgmma m64n256 into 128 fp32 registers per thread, then the epilogue straight from the fragments
// The epilogue stores pairs of neighbours: in the [i][j] layout two lanes (l, l ^ 4) swap one value so that each
// holds two consecutive j of one row; in the transposed [j][i] layout a thread's (b = 0, 1) values already are two
// consecutive i.  In the fp32 block every store instruction of a warp fills whole 32-byte sectors; in the fp16 block
// it writes 16 contiguous bytes per row.
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_MAX_STAGES = 8;

struct GemmParams {
    int E, Kp, bk, mma_k, kbs;
    long V2, nb, row_start;
    int tiles_j, tiles_i;          // 256 x 256 tiles
    long total_tiles;
    float *out;
    long stride_i, stride_e;
    int fisher_epochs;
    uint32_t stage_bytes;          // planes * (16384 + 32768)
    int stages;
    float out_scale;               // accumulator scale applied in the epilogue
    int tiled;                     // 1: output is tiled [tiles_i][tiles_j][E][256][256] fp32, 2: same in fp16;
                                   // 0: strided fp32 [i][e][j]
    // ---- symmetric (self-correlation) mode: corr[i][e][j] == corr[j][e][i], so a tile is computed once and stored
    // twice, as tile (ti, tj) and transposed as tile (tj, ti)
    long col_start;                // first column voxel of the block: column tile tj starts at col_start + 256*tj
    float *out_t;                  // tiled block [tiles_j - t_tj0][tiles_i][E][256 j][256 i] receiving the transposed
                                   // copy of every tile with tj >= t_tj0 (nullptr: none)
    int t_tj0;                     // column tiles [0, t_tj0) are the diagonal block (same voxels as the rows)
    int sym_diag;                  // 1: inside the diagonal block skip tiles tj < ti; tiles tj > ti are mirrored
                                   //    into `out` as tile (tj, ti)
    uint32_t bar_off;              // smem offset of the mbarriers
    int e_begin;                   // first epoch of this launch
};

// scale (+ Fisher-z) of the four accumulators of one n-block of a thread; the series form is taken for the warp's
// 8 x 16 block when no element exceeds its bound, else every element picks its form by its own value
__device__ __forceinline__ void epilogue_math4(float (&x)[4], float osc, bool do_fisher)
{
    if (!do_fisher) {
#pragma unroll
        for (int k = 0; k < 4; k++) x[k] = __fmaf_rn(x[k], osc, 0.f);
        return;
    }
    float m = 0.f;
#pragma unroll
    for (int k = 0; k < 4; k++) m = fmaxf(m, fabsf(x[k]));
    if (__any_sync(0xffffffffu, m * osc > FISHER_SERIES_MAX)) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float r = x[k] * osc;
            x[k] = fabsf(r) > FISHER_SERIES_MAX ? fisher_fast(r) : fisher_series1(r);
        }
    } else {
        const float2 a = fisher_series2(make_float2(x[0], x[1]), osc), b = fisher_series2(make_float2(x[2], x[3]), osc);
        x[0] = a.x, x[1] = a.y, x[2] = b.x, x[3] = b.y;
    }
}

template <bool HALF_OUT>
__device__ __forceinline__ void gemm_epilogue(const GemmParams &p, float (&acc)[128], int e, int tj, int ti, int half,
                                              int cw, int warp4, int lane)
{
    const int g = lane >> 2, qd = lane & 3, odd = g & 1;
    const int jl0 = half * 128 + cw * 64 + warp4 * 16 + g;   // j inside the 256 tile of h = 0 (h = 1: + 8)
    const bool do_fisher = e < p.fisher_epochs;
    const long i0 = (long)ti * 256;
    // where the transposed copy of this tile goes (tile-uniform; element offset into an fp32 or fp16 block)
    float *tbase = nullptr;
    size_t toff = 0;
    if (p.out_t != nullptr && tj >= p.t_tj0)
        tbase = p.out_t, toff = (((size_t)(tj - p.t_tj0) * p.tiles_i + ti) * p.E + e) * 65536;
    else if (p.sym_diag && tj > ti && tj < p.t_tj0)
        tbase = p.out, toff = (((size_t)tj * p.tiles_j + ti) * p.E + e) * 65536;
    const size_t tile_off = (((size_t)ti * p.tiles_j + tj) * p.E + e) * 65536;
#pragma unroll
    for (int n = 0; n < 32; n++) {
        if (i0 + ((8 * n) & ~31) >= p.nb) break;          // 32-row chunks past the block are not written
        float x[4] = {acc[4 * n], acc[4 * n + 1], acc[4 * n + 2], acc[4 * n + 3]};
        epilogue_math4(x, p.out_scale, do_fisher);
        const int il = 8 * n + 2 * qd;                   // rows il (b = 0) and il + 1 (b = 1)
        if (p.tiled) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const float v0 = x[2 * h], v1 = x[2 * h + 1];
                const float other = __shfl_xor_sync(0xffffffffu, odd ? v0 : v1, 4);
                // even g: (row il; columns j, j + 1), odd g: (row il + 1; columns j - 1, j)
                const size_t off = tile_off + (size_t)(il + odd) * 256 + (jl0 + 8 * h - odd);
                const float lo = odd ? other : v0, hi = odd ? v1 : other;
                if constexpr (HALF_OUT) {
                    *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(p.out) + off) = __floats2half2_rn(lo, hi);
                    if (tbase)
                        *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(tbase) + toff + (size_t)(jl0 + 8 * h) * 256 + il) =
                            __floats2half2_rn(v0, v1);
                } else {
                    // the block is far larger than L2 and is read back only by the next kernel: streaming stores keep
                    // the operand tiles (re-read by every tile of a column group) in L2
                    __stcs(reinterpret_cast<float2 *>(p.out + off), make_float2(lo, hi));
                    if (tbase) __stcs(reinterpret_cast<float2 *>(tbase + toff + (size_t)(jl0 + 8 * h) * 256 + il), make_float2(v0, v1));
                }
            }
        } else {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const long j = p.col_start + (long)tj * 256 + jl0 + 8 * h;
                if (j >= p.V2) continue;
                float *ptr = p.out + (size_t)e * p.stride_e + j + (size_t)(i0 + il) * p.stride_i;
                if (i0 + il < p.nb) ptr[0] = x[2 * h];
                if (i0 + il + 1 < p.nb) ptr[p.stride_i] = x[2 * h + 1];
            }
        }
    }
}

template <int FMT>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d)
{
    if constexpr (FMT == 0) wgmma_m64n256_f16(d, da, db, scale_d);
    else if constexpr (FMT == 1) wgmma_m64n256_bf16(d, da, db, scale_d);
    else wgmma_m64n256_tf32(d, da, db, scale_d);
}

// One k-block of a tile as one straight-line wgmma group: NK k-steps of every product, in prec_info's order (small cross
// terms first, hi * hi last; one product with one plane).  The fence and the commit are part of the batch: with them
// after the caller's switch on NK, ptxas closes a group at the end of each case and the commit adds an empty one.
template <int FMT, int PLANES, int NK>
__device__ __forceinline__ void corr_batch(float (&d)[128], uint32_t cols, uint32_t rows, uint32_t scale_first)
{
    constexpr int SEGS = PLANES == 2 ? 3 : 1;
    wgmma_fence();
#pragma unroll
    for (int sgm = 0; sgm < SEGS; sgm++) {
        const int pc = PLANES == 2 && sgm == 1, pr = PLANES == 2 && sgm == 0;   // seg_c {0, 1, 0}, seg_r {1, 0, 0}
        const uint64_t da = make_wgmma_desc_sw128(cols + pc * 16384);
        const uint64_t db = make_wgmma_desc_sw128(rows + pr * 32768);
#pragma unroll
        for (int k = 0; k < NK; k++) wgmma_m64n256<FMT>(d, da + 2 * k, db + 2 * k, sgm == 0 && k == 0 ? scale_first : 1u);
    }
    wgmma_commit();
}

// tile t of this launch -> (epoch, column tile, row tile); false: a mirrored tile of the symmetric diagonal block
__device__ __forceinline__ bool gemm_tile_coords(const GemmParams &p, long tile, int &e, int &tj, int &ti)
{
    const long tiles_per_e = (long)p.tiles_j * p.tiles_i;
    const int el = (int)(tile / tiles_per_e);
    const long rem = tile - (long)el * tiles_per_e;
    e = p.e_begin + el;
    tj = (int)(rem / p.tiles_i);
    ti = (int)(rem - (long)tj * p.tiles_i);
    return !(p.sym_diag && tj < ti);
}

template <int FMT, int PLANES, bool HALF_OUT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    k_corr_wgmma(const __grid_constant__ CUtensorMap tm_cols, const __grid_constant__ CUtensorMap tm_rows,
                 const GemmParams p)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + p.bar_off);   // [stages] TMA bytes landed
    uint64_t *empty_bar = full_bar + GEMM_MAX_STAGES;                       // [stages] both consumer warpgroups done

    const int warp = uniform_warp_idx();
    const int wg = warp >> 2;
    const int lane = threadIdx.x & 31;
    const int half = (int)(blockIdx.x & 1);
    const long pair = blockIdx.x >> 1, npairs = gridDim.x >> 1;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_cols);
        tma_prefetch_desc(&tm_rows);
        for (int s = 0; s < p.stages; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 256);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one_sync()) {
            int stage = 0;
            uint32_t phase = 0;
            for (long tile = pair; tile < p.total_tiles; tile += npairs) {
                int e, tj, ti;
                if (!gemm_tile_coords(p, tile, e, tj, ti)) continue;
                const int col0 = (int)p.col_start + tj * 256 + half * 128;
                const int row0 = (int)(p.row_start + (long)ti * 256);
                for (int kb = 0; kb < p.kbs; kb++) {
                    const int k0 = kb * p.bk;
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], p.stage_bytes);
                    uint8_t *base = smem + (size_t)stage * p.stage_bytes;
                    for (int pl = 0; pl < PLANES; pl++) {
                        tma_load_3d(&tm_cols, &full_bar[stage], base + pl * 16384, k0, col0, pl * p.E + e);
                        tma_load_3d(&tm_rows, &full_bar[stage], base + PLANES * 16384 + pl * 32768, k0, row0,
                                    pl * p.E + e);
                    }
                    if (++stage == p.stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ wgmma + epilogue
        setmaxnreg_inc<232>();
        const int cw = wg - 1;             // consumer warpgroup: columns 64 cw .. of the CTA's 128
        const uint32_t tiles_addr = smem_u32(smem);
        int stage = 0;
        uint32_t phase = 0;
        float acc[128];
#pragma unroll
        for (int k = 0; k < 128; k++) acc[k] = 0.f;
        for (long tile = pair; tile < p.total_tiles; tile += npairs) {
            int e, tj, ti;
            if (!gemm_tile_coords(p, tile, e, tj, ti)) continue;
            for (int kb = 0; kb < p.kbs; kb++) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t base = tiles_addr + (uint32_t)stage * p.stage_bytes;
                const uint32_t cols = base + cw * 8192, rows = base + PLANES * 16384;
                const int rem_k = p.Kp - kb * p.bk;
                const uint32_t scale_first = kb > 0;
                switch ((rem_k < p.bk ? rem_k : p.bk) / p.mma_k) {   // bk / mma_k == 4 for every format: 32 B per k-step
                case 1: corr_batch<FMT, PLANES, 1>(acc, cols, rows, scale_first); break;
                case 2: corr_batch<FMT, PLANES, 2>(acc, cols, rows, scale_first); break;
                case 3: corr_batch<FMT, PLANES, 3>(acc, cols, rows, scale_first); break;
                default: corr_batch<FMT, PLANES, 4>(acc, cols, rows, scale_first); break;
                }
                wgmma_wait_all();
                mbar_arrive(&empty_bar[stage]);
                if (++stage == p.stages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            gemm_epilogue<HALF_OUT>(p, acc, e, tj, ti, half, cw, warp & 3, lane);
        }
    }
}


// ---------------------------------------------------------------- tensor-map creation (driver entry point)
typedef CUresult (*PFN_tmEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                      const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                      CUtensorMapFloatOOBfill);
static PFN_tmEncodeTiled get_encode_fn()
{
    static PFN_tmEncodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_tmEncodeTiled>(p);
        else
            cudaGetLastError();
    });
    return fn;
}

// operand tensor [planes*E][V][Kp] (Kp fastest), box = {bk, rows, 1}, 128-byte swizzle, zero OOB fill
static int make_operand_map(CUtensorMap *m, const void *base, const PrecInfo &pi, int E, long V, int Kp,
                            int box_rows)
{
    PFN_tmEncodeTiled enc = get_encode_fn();
    if (!enc) return fail(FCMA_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[3] = {(cuuint64_t)Kp, (cuuint64_t)V, (cuuint64_t)pi.planes * E};
    cuuint64_t gstr[2] = {(cuuint64_t)Kp * pi.esize, (cuuint64_t)V * Kp * pi.esize};
    cuuint32_t box[3] = {(cuuint32_t)pi.bk, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMapDataType dt = pi.pack == 0 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                             : pi.pack == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUresult r = enc(m, dt, 3, const_cast<void *>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(FCMA_ECUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return FCMA_OK;
}


// tiled block [ntg tile groups][E][256 i][256 j] (fp32 or fp16) as the 5-D tensor the TMA column pass reads:
// (j, i%4, tile group * E/4 + e/4, (i%256)/4, e%4), box = one brick (32, 4, 8, 4, 4); see k_norm_syrk_cols_tma
static int make_cols_map(CUtensorMap *m, const void *base, size_t ntg, int E, int half_in)
{
    PFN_tmEncodeTiled enc = get_encode_fn();
    if (!enc) return fail(FCMA_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    const cuuint64_t esz = half_in ? 2 : 4;
    cuuint64_t gdim[5] = {256, 4, (cuuint64_t)ntg * (cuuint64_t)(E / 4), 64, 4};
    cuuint64_t gstr[4] = {256 * esz, 4 * 65536 * esz, 4 * 256 * esz, 65536 * esz};
    cuuint32_t box[5] = {32, 4, 8, 4, 4};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(m, half_in ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5,
                     const_cast<void *>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     half_in ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(FCMA_ECUDA, "cuTensorMapEncodeTiled (column pass) failed with CUresult %d", (int)r);
    return FCMA_OK;
}

// self-correlation fix-up: out[i][e][start+i] = exact sequential-FMA r (optionally Fisher-transformed)
__global__ void k_self_corr_fixup(const float *__restrict__ selfdiag, int E, long V, long start, long nb, float *out,
                                  long stride_i, long stride_e, int fisher_epochs, long tiled_t256, int half_out,
                                  long col_start)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nb * E) return;
    const long i = idx / E;
    const int e = (int)(idx - i * E);
    float r = selfdiag[(size_t)e * V + start + i];
    if (e < fisher_epochs) r = fisher_fast(r);
    const long j = start + i - col_start;   // column inside the block
    if (tiled_t256 > 0) {   // tiled [i/256][j/256][e][i%256][j%256], fp32 or fp16 elements
        const size_t off = ((((size_t)(i >> 8) * tiled_t256 + (j >> 8)) * E + e) * 256 + (i & 255)) * 256 + (j & 255);
        if (half_out)
            reinterpret_cast<__half *>(out)[off] = __float2half_rn(r);
        else
            out[off] = r;
    } else {
        out[(size_t)i * stride_i + (size_t)e * stride_e + j] = r;
    }
}

// tiled_t256 > 0: write the block in the tiled layout [ceil(nb/256)][tiled_t256][E][256][256] (the caller
// provides round_up(nb, 256) rows of workspace and tiled_t256 == ceil(V2/256)); else out[i*stride_i + e*stride_e + j]
// Symmetric mode (sym != nullptr; self-correlation, tiled fp32 output): the block covers columns [col_start, V2)
// with col_start == start; column tiles below t_tj0 = ceil(nb/256) are the diagonal block, where only tiles
// tj >= ti are computed and tiles tj > ti are mirrored into `out`; every tile with tj >= t_tj0 is also stored
// transposed into sym->out_t, a tiled block [tiles_j - t_tj0][ceil(nb/256)][E][256][256] (rows = the column voxels).
struct SymOut {
    float *out_t;      // nullptr: no transposed block (the column-direction pass reads block A instead)
};
static int launch_corr_mma(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                           long start, long nb, float *out, long stride_i, long stride_e, int fisher_epochs,
                           cudaStream_t st, long tiled_t256 = 0, int half_out = 0, const SymOut *sym = nullptr,
                           int e_begin = 0, int e_count = -1, bool fixup = true)
{
    PrecInfo pi;
    if (!prec_info(precision, &pi)) return fail(FCMA_EINVAL, "unknown precision %d", precision);
    if (E <= 0 || T <= 0 || V <= 0 || V2 <= 0 || nb <= 0 || start < 0 || start + nb > V)
        return fail(FCMA_EINVAL, "bad shape E=%d T=%d V=%ld V2=%ld start=%ld nb=%ld", E, T, V, V2, start, nb);
    if (((uintptr_t)rows_op & 15) || ((uintptr_t)cols_op & 15))
        return fail(FCMA_EINVAL, "packed operands must be 16-byte aligned");
    if (V >= (1L << 31) || V2 >= (1L << 31) || nb >= (1L << 31))
        return fail(FCMA_EINVAL, "voxel count exceeds TMA coordinate range");
    const int Kp = fcma_operand_kp(precision, T);

    GemmParams q;
    memset(&q, 0, sizeof(q));
    q.E = E, q.Kp = Kp, q.bk = pi.bk, q.mma_k = pi.mma_k, q.kbs = (int)cdiv(Kp, pi.bk);
    q.V2 = V2, q.nb = nb, q.row_start = start;
    q.col_start = sym ? start : 0;
    q.tiles_j = (int)cdiv(V2 - q.col_start, 256), q.tiles_i = (int)cdiv(nb, 256);
    if (sym) {
        if (rows_op != cols_op || V != V2 || tiled_t256 <= 0 || ((nb & 255) && start + nb != V))
            return fail(FCMA_EINVAL, "internal: symmetric GEMM needs self-correlation, the tiled block and whole row tiles");
        q.sym_diag = 1;
        q.t_tj0 = q.tiles_i;
        q.out_t = q.tiles_j > q.tiles_i ? sym->out_t : nullptr;
    }
    if (e_count < 0) e_count = E - e_begin;
    if (e_begin < 0 || e_count <= 0 || e_begin + e_count > E) return fail(FCMA_EINVAL, "internal: bad epoch range [%d, +%d) of %d", e_begin, e_count, E);
    q.e_begin = e_begin;
    q.total_tiles = (long)q.tiles_j * q.tiles_i * e_count;
    q.out = out, q.stride_i = stride_i, q.stride_e = stride_e, q.fisher_epochs = fisher_epochs;
    q.out_scale = 1.0f / (pi.in_scale * pi.in_scale);
    q.stage_bytes = (uint32_t)pi.planes * (16384 + 32768);
    q.tiled = tiled_t256 > 0 ? (half_out ? 2 : 1) : 0;
    if (half_out && !q.tiled) return fail(FCMA_EINVAL, "internal: fp16 output needs the tiled layout");
    if (q.tiled && tiled_t256 != q.tiles_j) return fail(FCMA_EINVAL, "internal: tiled output needs T256 == tiles_j");
    const size_t cap = 227 * 1024 - 1024 /*alignment slack*/ - 256 /*barriers*/;
    int stages = (int)(cap / q.stage_bytes);
    if (stages > GEMM_MAX_STAGES) stages = GEMM_MAX_STAGES;
    {
        const char *sg = diag_env("FCMA_GEMM_STAGES");         // A/B: cap the number of smem stages
        if (sg && atoi(sg) >= 2 && atoi(sg) < stages) stages = atoi(sg);
    }
    if (stages < 2) return fail(FCMA_EINVAL, "internal: not enough shared memory for 2 stages");
    q.stages = stages;
    q.bar_off = (uint32_t)((size_t)stages * q.stage_bytes);
    const size_t smem = (size_t)stages * q.stage_bytes + 1024 + 256;

    CUtensorMap tm_cols, tm_rows;
    int rc = make_operand_map(&tm_cols, cols_op, pi, E, V2, Kp, 128);
    if (rc) return rc;
    rc = make_operand_map(&tm_rows, rows_op, pi, E, V, Kp, 256);
    if (rc) return rc;

    // persistent grid: two CTAs (the two column halves) per 256 x 256 tile, one CTA per SM
    long pairs = g_sm_count / 2;
    if (q.total_tiles < pairs) pairs = q.total_tiles;
    {
        // diagnostic build: FCMA_GEMM_PAIRS=n caps the persistent grid at n CTA pairs, leaving SMs to kernels of another
        // stream
        const char *gp = diag_env("FCMA_GEMM_PAIRS");
        if (gp && atoi(gp) >= 1 && atoi(gp) < pairs) pairs = atoi(gp);
    }
    auto gemm = [&](auto kernel) {
        rc = launch_kernel(kernel, (unsigned)(2 * pairs), GEMM_THREADS, smem, st, "k_corr_wgmma", tm_cols, tm_rows, q);
    };
    // the kernel compiles the product order in (corr_batch): one product with one plane, prec_info's three with two
    const bool order_ok = pi.planes == 1 ? pi.segs == 1
                                         : pi.segs == 3 && pi.seg_r[0] == 1 && pi.seg_r[1] == 0 && pi.seg_r[2] == 0 &&
                                               pi.seg_c[0] == 0 && pi.seg_c[1] == 1 && pi.seg_c[2] == 0;
    auto go = [&](auto FMT, auto PLANES) {
        half_out ? gemm(k_corr_wgmma<FMT, PLANES, true>) : gemm(k_corr_wgmma<FMT, PLANES, false>);
    };
    if (!order_ok) return fail(FCMA_EINVAL, "internal: k_corr_wgmma has no product order for precision %d", precision);
    if (pi.fmt == 0 && pi.planes == 2) go(IntC<0>{}, IntC<2>{});        // fp16x3
    else if (pi.fmt == 1 && pi.planes == 1) go(IntC<1>{}, IntC<1>{});   // bf16
    else if (pi.fmt == 1 && pi.planes == 2) go(IntC<1>{}, IntC<2>{});   // bf16x3
    else if (pi.fmt == 2 && pi.planes == 1) go(IntC<2>{}, IntC<1>{});   // tf32
    else if (pi.fmt == 2 && pi.planes == 2) go(IntC<2>{}, IntC<2>{});   // tf32x3
    else return fail(FCMA_EINVAL, "internal: no k_corr_wgmma instantiation for operand type %d, %d planes", pi.fmt, pi.planes);
    if (rc) return rc;

    if (rows_op == cols_op && V == V2 && fixup) {
        // self-correlation: replace the diagonal by the reference-exact values kept with the operand
        const float *sd = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(rows_op) +
                                                          operand_plane_bytes(pi, precision, E, T, V));
        long n = nb * E;
        k_self_corr_fixup<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(sd, E, V, start, nb, out, stride_i, stride_e,
                                                                 fisher_epochs, tiled_t256, half_out, q.col_start);
        LAUNCH_CHECK("k_self_corr_fixup");
    }
    return FCMA_OK;
}

// ============================================================================================
// a4 reference-order path: fp32 FFMA tiled GEMM on the raw epochs [E][T][ld]
// ============================================================================================
// out[i][e][j] = sum_t R[e][t][start+i] * C[e][t][j];  64x64 tile, 256 threads, 4x4 micro-tile
__global__ void __launch_bounds__(256) k_corr_simt(const float *__restrict__ R, long ldr, const float *__restrict__ C,
                                                   long ldc, int T, long V2, long start, long nb, float *out,
                                                   long stride_i, long stride_e)
{
    __shared__ float sr[16][64 + 4];
    __shared__ float sc[16][64 + 4];
    const int e = blockIdx.z;
    const long i0 = (long)blockIdx.y * 64, j0 = (long)blockIdx.x * 64;
    const float *Re = R + (size_t)e * T * ldr;
    const float *Ce = C + (size_t)e * T * ldc;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int t0 = 0; t0 < T; t0 += 16) {
        for (int idx = threadIdx.x; idx < 16 * 64; idx += 256) {
            int tt = idx >> 6, x = idx & 63;
            int t = t0 + tt;
            long i = i0 + x, j = j0 + x;
            sr[tt][x] = (t < T && i < nb) ? Re[(size_t)t * ldr + start + i] : 0.f;
            sc[tt][x] = (t < T && j < V2) ? Ce[(size_t)t * ldc + j] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int tt = 0; tt < 16; tt++) {
            float a[4], b[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                a[k] = sr[tt][ty * 4 + k];
                b[k] = sc[tt][tx * 4 + k];
            }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) acc[x][y] = fmaf(a[x], b[y], acc[x][y]);
        }
        __syncthreads();
    }
    for (int x = 0; x < 4; x++) {
        long i = i0 + ty * 4 + x;
        if (i >= nb) continue;
        for (int y = 0; y < 4; y++) {
            long j = j0 + tx * 4 + y;
            if (j < V2) out[(size_t)i * stride_i + (size_t)e * stride_e + j] = acc[x][y];
        }
    }
}

// plain NT GEMM  C[m][n] = sum_k A[m][k] B[n][k]  (a12 / a15), K contiguous in both operands
__global__ void __launch_bounds__(256) k_gemm_nt(const float *__restrict__ A, const float *__restrict__ B, float *C,
                                                 long M, long N, long K, long lda, long ldb, long ldc)
{
    __shared__ float sa[64][16 + 1];
    __shared__ float sb[64][16 + 1];
    const long m0 = (long)blockIdx.y * 64, n0 = (long)blockIdx.x * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (long k0 = 0; k0 < K; k0 += 16) {
        for (int idx = threadIdx.x; idx < 64 * 16; idx += 256) {
            int r = idx >> 4, kk = idx & 15;
            long k = k0 + kk;
            sa[r][kk] = (k < K && m0 + r < M) ? A[(size_t)(m0 + r) * lda + k] : 0.f;
            sb[r][kk] = (k < K && n0 + r < N) ? B[(size_t)(n0 + r) * ldb + k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
            float a[4], b[4];
#pragma unroll
            for (int x = 0; x < 4; x++) {
                a[x] = sa[ty * 4 + x][kk];
                b[x] = sb[tx * 4 + x][kk];
            }
#pragma unroll
            for (int x = 0; x < 4; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) acc[x][y] = fmaf(a[x], b[y], acc[x][y]);
        }
        __syncthreads();
    }
    for (int x = 0; x < 4; x++) {
        long m = m0 + ty * 4 + x;
        if (m >= M) continue;
        for (int y = 0; y < 4; y++) {
            long n = n0 + tx * 4 + y;
            if (n < N) C[(size_t)m * ldc + n] = acc[x][y];
        }
    }
}

// util.py:32-60 on rows: zscore(axis=1, ddof=0), optional nan->0, / sqrt(D)
__global__ void __launch_bounds__(256) k_row_normalize(float *X, long R, long D, long ld, int nan_to_zero)
{
    __shared__ double s_red[256];
    __shared__ float s_val[2];
    for (long r = blockIdx.x; r < R; r += gridDim.x) {
        float *row = X + (size_t)r * ld;
        double s = 0.0;
        for (long d = threadIdx.x; d < D; d += 256) s += row[d];
        s_red[threadIdx.x] = s;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) s_val[0] = (float)(s_red[0] / D);
        __syncthreads();
        float mean = s_val[0];
        double q = 0.0;
        for (long d = threadIdx.x; d < D; d += 256) {
            float dd = row[d] - mean;
            q += (double)dd * dd;
        }
        __syncthreads();
        s_red[threadIdx.x] = q;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) s_val[1] = (float)sqrt(s_red[0] / D);
        __syncthreads();
        float sd = s_val[1];
        float rs = sqrtf((float)D);
        for (long d = threadIdx.x; d < D; d += 256) {
            float z = (row[d] - mean) / sd;  // sd==0 -> nan/inf as numpy
            if (nan_to_zero) {
                if (!(z == z)) z = 0.f;
                else if (isinf(z)) z = z > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
            }
            row[d] = z / rs;
        }
        __syncthreads();
    }
}

// ============================================================================================
// a6 standalone: exact restatement of fcma_extension.cc:52-84 (sequential fp32, no FMA contraction)
// ============================================================================================
// Fisher-z and z-score, in place, of subject s's epochs [s*eps, (s+1)*eps) of one column: mat[b * ld] is epoch b.  The one
// copy of this arithmetic: k_within_subject_norm and k_norm_gram_f64 (the per-voxel fp64 kernels of VoxelSelector's
// feature path) both call it, so their z values are bit-identical.
__device__ __forceinline__ void within_subject_column(float *mat, long ld, long s, int eps)
{
    float mean = 0.0f, sq = 0.0f;
    for (long b = s * eps; b < (s + 1) * eps; b++) {
        float r = mat[(size_t)b * ld];
        float num = __fadd_rn(1.0f, r);
        float den = __fsub_rn(1.0f, r);
        num = (num <= 0.0f) ? 1e-4f : num;
        den = (den <= 0.0f) ? 1e-4f : den;
        float z = __fmul_rn(0.5f, logf(__fdiv_rn(num, den)));
        mat[(size_t)b * ld] = z;
        mean = __fadd_rn(mean, z);
        sq = __fadd_rn(sq, __fmul_rn(z, z));
    }
    mean = __fdiv_rn(mean, (float)eps);
    float var = __fsub_rn(__fdiv_rn(sq, (float)eps), __fmul_rn(mean, mean));
    float inv = (var <= 0.0f) ? 0.0f : __fdiv_rn(1.0f, __fsqrt_rn(var));
    for (long b = s * eps; b < (s + 1) * eps; b++)
        mat[(size_t)b * ld] = __fmul_rn(__fsub_rn(mat[(size_t)b * ld], mean), inv);
}

__global__ void __launch_bounds__(256) k_within_subject_norm(float *data, long n0, int E, long n2, int eps)
{
    const long nSubjs = E / eps;
    const long total = n0 * nSubjs * n2;
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const long j = idx % n2;
        const long v = idx / n2;
        const long s = v % nSubjs;
        const long i = v / nSubjs;
        within_subject_column(data + (size_t)i * E * n2 + j, n2, s, eps);
    }
}

// ============================================================================================
// a7 standalone, fp32 FFMA: K_i = Z_i Z_i^T (any E), one block per voxel row
// ============================================================================================
__global__ void __launch_bounds__(256) k_syrk_simt(const float *__restrict__ z, long nb, int E, long n2, long stride_i,
                                                   long ld, float beta, float *K, int sum_over_rows)
{
    extern __shared__ float s_z[];  // [64 j][E+1]
    const int EP = E + 1;
    for (long i = blockIdx.x; i < nb; i += gridDim.x) {
        const float *zi = z + (size_t)i * stride_i;
        const int npairs = E * E;
        // each thread owns pairs tid, tid+256, ... (at most 16 for E <= 64; loop for larger E)
        for (int pbase = 0; pbase < npairs; pbase += 256 * 16) {
            float acc[16];
#pragma unroll
            for (int k = 0; k < 16; k++) acc[k] = 0.f;
            for (long j0 = 0; j0 < n2; j0 += 64) {
                __syncthreads();
                for (int idx = threadIdx.x; idx < E * 64; idx += 256) {
                    int e = idx >> 6, jj = idx & 63;
                    s_z[jj * EP + e] = (j0 + jj < n2) ? zi[(size_t)e * ld + j0 + jj] : 0.f;
                }
                __syncthreads();
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    int pidx = pbase + k * 256 + threadIdx.x;
                    if (pidx < npairs) {
                        int a = pidx / E, b = pidx - a * E;
                        float s = acc[k];
                        for (int jj = 0; jj < 64; jj++) s = fmaf(s_z[jj * EP + a], s_z[jj * EP + b], s);
                        acc[k] = s;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < 16; k++) {
                int pidx = pbase + k * 256 + threadIdx.x;
                if (pidx < npairs) {
                    if (sum_over_rows) {
                        atomicAdd(&K[pidx], acc[k]);
                    } else {
                        float *dst = &K[(size_t)i * npairs + pidx];
                        *dst = (beta == 0.f ? 0.f : beta * *dst) + acc[k];
                    }
                }
            }
        }
    }
}

// ============================================================================================
// a6+a7 fused on warp MMAs: Fisher-z, within-subject z-score and K_i = Z_i Z_i^T in one pass
// over the correlation block; the normalised values never leave registers.
// ============================================================================================
// z-score coefficients of a subject (two columns at once) from the sums of its EPS values and of their squares:
// z = x * inv + mi.  nm = -mean, negvar = mean^2 - E[x^2] (both exact rescalings: EPS is a power of two); a variance
// <= 0 gives inv = 0, so a constant subject normalises to zeros.
template <int EPS>
__device__ __forceinline__ void subject_coeffs(float2 msum, float2 s2sum, float2 &inv, float2 &mi)
{
    const float2 nm = ffma2(msum, splat2(-1.0f / EPS), splat2(0.f));
    const float2 ns2 = ffma2(s2sum, splat2(-1.0f / EPS), splat2(0.f));
    const float2 negvar = neg_variance<EPS>(nm, ns2);
    inv.x = negvar.x >= 0.f ? 0.f : rsqrt_ftz(-negvar.x);
    inv.y = negvar.y >= 0.f ? 0.f : rsqrt_ftz(-negvar.y);
    mi = ffma2(nm, inv, splat2(0.f));
}

// Within-subject z-score of the values a lane holds in mma-fragment layout: epochs R*g + r (r < R) x NS slots x NU
// columns, element v(r, s, u), two adjacent columns per packed fp32x2 op.  The epochs of one subject (EPS, a power of
// two) lie inside the lane when EPS <= R, otherwise in EPS/R adjacent g-lanes (xor shuffles over lanes 4o).  Only
// epochs of complete subjects (< S_eps) change.  The subject group is the outermost loop: moving it inside the
// (slot, column) loops changes the kernels' instruction mix and spills.  all_valid (block-uniform, every real epoch in a
// complete subject; padded epochs hold zeros and normalise to zeros) lets the shuffle path skip the per-lane select.
template <int EPS, int R, int NS, int NU, typename V>
__device__ __forceinline__ void zscore_frag(V &&v, int g, int S_eps, bool all_valid = false)
{
    auto apply = [&](int r, int s, int u, float2 inv, float2 mi) {
        const float2 z = ffma2(make_float2(v(r, s, u), v(r, s, u + 1)), inv, mi);
        v(r, s, u) = z.x, v(r, s, u + 1) = z.y;
    };
    if constexpr (EPS <= R) {
#pragma unroll
        for (int q = 0; q < R / EPS; q++) {
            const bool valid = R * g + q * EPS < S_eps;
#pragma unroll
            for (int s = 0; s < NS; s++)
#pragma unroll
                for (int u = 0; u < NU; u += 2) {
                    float2 m = splat2(0.f), s2 = splat2(0.f);
#pragma unroll
                    for (int b = 0; b < EPS; b++) {
                        const float2 x = make_float2(v(q * EPS + b, s, u), v(q * EPS + b, s, u + 1));
                        m = ffma2(x, splat2(1.f), m);
                        s2 = ffma2(x, x, s2);
                    }
                    float2 inv, mi;
                    subject_coeffs<EPS>(m, s2, inv, mi);
                    if (valid) {
#pragma unroll
                        for (int b = 0; b < EPS; b++) apply(q * EPS + b, s, u, inv, mi);
                    }
                }
        }
    } else {
        constexpr int L = EPS / R;   // adjacent g-lanes per subject
        const bool valid = R * g < S_eps;
#pragma unroll
        for (int s = 0; s < NS; s++)
#pragma unroll
            for (int u = 0; u < NU; u += 2) {
                float2 m = splat2(0.f), s2 = splat2(0.f);
#pragma unroll
                for (int r = 0; r < R; r++) {
                    const float2 x = make_float2(v(r, s, u), v(r, s, u + 1));
                    m = ffma2(x, splat2(1.f), m);
                    s2 = ffma2(x, x, s2);
                }
#pragma unroll
                for (int o = 1; o < L; o <<= 1) {
                    m.x += __shfl_xor_sync(0xffffffffu, m.x, 4 * o);
                    m.y += __shfl_xor_sync(0xffffffffu, m.y, 4 * o);
                    s2.x += __shfl_xor_sync(0xffffffffu, s2.x, 4 * o);
                    s2.y += __shfl_xor_sync(0xffffffffu, s2.y, 4 * o);
                }
                float2 inv, mi;
                subject_coeffs<EPS>(m, s2, inv, mi);
                if (all_valid) {   // uniform branch: no per-value select
#pragma unroll
                    for (int r = 0; r < R; r++) apply(r, s, u, inv, mi);
                } else if (valid) {
#pragma unroll
                    for (int r = 0; r < R; r++) apply(r, s, u, inv, mi);
                }
            }
    }
}

// One block (8 warps) per voxel row i; warps stride over 32-column chunks of the [E][n2] slab.
// Lane (g = lane/4, t = lane%4) loads, as float4s, epochs R*g .. R*g+R-1 at columns
// j0 + 16h + 4t .. +3 (h = 0,1).  These registers are at once
//   - the A fragments (rows g, g+8 of m-tile mu <-> epochs R*g+2mu, R*g+2mu+1) and
//   - the B fragments (col g of n-tile nu <-> epoch R*g+nu)
// of mma.sync.m16n8k8 (tf32), with k-slots t / t+4 <-> two adjacent columns of the lane (see the MMA loop) for
// k-step u = 0..3: a sum over columns is invariant under that permutation, and the epoch
// permutation is undone when the accumulators are scattered.  EP = 8R padded epochs.
// The epochs of one subject (EPS consecutive epochs, EPS a power of two) live in EPS/R adjacent
// g-lanes (or inside a lane when EPS <= R), so the z-score statistics need at most 3 shuffles.
// EPS == 0: input is already normalised (plain SYRK).
// VEC: 0 scalar loads (unaligned fp32 block), 1 cp.async of an fp32 block, 2 cp.async of an fp16 block (tiled
// intermediate written by the GEMM epilogue; a lane then takes 8 consecutive columns 8t..8t+7 per epoch as ONE
// 16-byte copy -- which columns a k-slot stands for is irrelevant to a sum over columns).
// EPS > 0: the z-scored values feed mma.m16n8k16 (fp16); EPS == 0 (already normalised input) keeps mma.m16n8k8 (tf32).
template <int R, int EPS, bool FISHER, int VEC>
__global__ void __launch_bounds__(256, (R <= 4 ? 2 : 1))
    k_norm_syrk(const float *__restrict__ C, long nb, int E, long n2, long stride_i, long ld, long chunk_step,
                long self_col0, float beta, float *K, int sum_over_rows, long rb_stride, double *K64)
{
    constexpr int EP = 8 * R;
    constexpr int MT = EP / 16, NT = EP / 8;
    __shared__ float s_K[EP * EP];
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    float4 *s_stage = reinterpret_cast<float4 *>(dyn_smem);  // VEC only: [warp][buf][copy][lane]
    // R <= 4 only: per-warp fp32 partial kernels [8][EP*EP].  The warp MMA adds into its accumulator
    // with truncation, so a long chain at growing magnitude biases the sums (measured 5e-5 relative on
    // the diagonal at V2 = 50 000); flushing the MMA accumulators into these round-to-nearest partials
    // every FLUSH chunks bounds the chain length (bias ~1e-6).  Every (row, col) has exactly one owner lane.
    constexpr int CPL = VEC == 2 ? R : 2 * R;   // 16-byte copies per lane and chunk
    using elem_t = std::conditional_t<VEC == 2, __half, float>;
    [[maybe_unused]] float *s_part =
        reinterpret_cast<float *>(dyn_smem + (VEC ? (size_t)8 * 2 * CPL * 32 * sizeof(float4) : 0));
    constexpr int FLUSH = 8;   // chunks between flushes of the MMA accumulators (bounds the truncating accumulation chain)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = EPS > 0 ? (E / EPS) * EPS : 0;  // epochs that get normalised
    const long nchunks = (n2 + 31) / 32;

    for (long i = blockIdx.x; i < nb; i += gridDim.x) {
        // classic layout: row i at i*stride_i; tiled layout (chunk_step != 256): 256-row blocks of
        // ceil(n2/256) * chunk_step floats, rows 256 floats apart inside a block
        const elem_t *Cb = reinterpret_cast<const elem_t *>(C);
        const elem_t *Ci = chunk_step == 256
                               ? Cb + (size_t)i * stride_i
                               : Cb + (size_t)(i >> 8) * (size_t)(rb_stride ? rb_stride : ((n2 + 255) >> 8) * chunk_step) +
                                     (size_t)(i & 255) * stride_i;
        const long self_col = self_col0 >= 0 ? self_col0 + i : -1;
        float acc[MT][NT][4];
#pragma unroll
        for (int a = 0; a < MT; a++)
#pragma unroll
            for (int b = 0; b < NT; b++)
#pragma unroll
                for (int c = 0; c < 4; c++) acc[a][b][c] = 0.f;

        [[maybe_unused]] int since_flush = 0;
        auto flush = [&]() {
            float *part = s_part + warp * (EP * EP);
#pragma unroll
            for (int mu = 0; mu < MT; mu++)
#pragma unroll
                for (int nu = 0; nu < NT; nu++) {
                    const int row0 = R * g + 2 * mu, row1 = row0 + 1;
                    const int col0 = R * (2 * t) + nu, col1 = R * (2 * t + 1) + nu;
                    part[row0 * EP + col0] += acc[mu][nu][0];
                    part[row0 * EP + col1] += acc[mu][nu][1];
                    part[row1 * EP + col0] += acc[mu][nu][2];
                    part[row1 * EP + col1] += acc[mu][nu][3];
#pragma unroll
                    for (int c = 0; c < 4; c++) acc[mu][nu][c] = 0.f;
                }
        };
        // R == 8: the block's s_K is kept in FRAGMENT order, element ((mu*NT + nu)*4 + c)*32 + lane, so that the 32 lanes
        // of an atomic instruction hit 32 different banks (in (row, col) order they collide 16-way: rows 8g.. are 512
        // floats apart); frag_index() below maps (row, col) back when the row is written out.
        auto flush_atomic = [&]() {
#pragma unroll
            for (int mu = 0; mu < MT; mu++)
#pragma unroll
                for (int nu = 0; nu < NT; nu++) {
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        atomicAdd(&s_K[((mu * NT + nu) * 4 + c) * 32 + lane], acc[mu][nu][c]);
                        acc[mu][nu][c] = 0.f;
                    }
                }
        };
        // (row, col) of the padded EP x EP matrix -> position in fragment order: row = R*g + 2*mu + (c >> 1),
        // col = R*(2*t + (c & 1)) + nu, lane = 4*g + t
        [[maybe_unused]] auto frag_index = [](int row, int col) {
            const int gg = row / R, mu = (row % R) >> 1, ch = row & 1;
            const int q = col / R, nu = col % R, tt = q >> 1, cl = q & 1;
            return ((mu * NT + nu) * 4 + (ch * 2 + cl)) * 32 + 4 * gg + tt;
        };
        if constexpr (R <= 4) {
            float *part = s_part + warp * (EP * EP);
            for (int idx = lane; idx < EP * EP; idx += 32) part[idx] = 0.f;
            __syncwarp();
        } else {
            for (int idx = threadIdx.x; idx < EP * EP; idx += 256) s_K[idx] = 0.f;
            __syncthreads();
        }
        // VEC path: cp.async double buffering into a per-warp staging tile (8 x 16 B per lane), so the
        // next chunk streams from HBM while this one is normalised and multiplied; zero fill covers
        // epochs >= E and the ragged last chunk without any branch.
        [[maybe_unused]] float4 *stage = nullptr;
        [[maybe_unused]] const elem_t *lane_src[R];  // row pointers of this lane, advanced chunk by chunk
        [[maybe_unused]] uint32_t row_bytes[R];      // 16 for epochs < E, 0 (-> zero fill) otherwise
        [[maybe_unused]] int buf = 0;
        // issue the CPL 16-byte copies of the chunk starting at column jc into staging buffer b
        auto prefetch = [&](long jc, int b) {
            float4 *dst = stage + b * (CPL * 32) + lane;
            if constexpr (VEC == 2) {
                if (jc + 32 <= n2) {  // warp-uniform: full chunk
#pragma unroll
                    for (int r = 0; r < R; r++) cp_async_16_zfill(dst + r * 32, lane_src[r], row_bytes[r]);
                } else {
#pragma unroll
                    for (int r = 0; r < R; r++) {
                        long left = (n2 - (jc + 8 * t)) * 2;
                        uint32_t nbytes = left <= 0 ? 0u : (left < 16 ? (uint32_t)left : 16u);
                        nbytes = row_bytes[r] ? nbytes : 0u;
                        cp_async_16_zfill(dst + r * 32, nbytes ? lane_src[r] : Ci, nbytes);
                    }
                }
            } else {
                if (jc + 32 <= n2) {  // warp-uniform: full chunk
#pragma unroll
                    for (int r = 0; r < R; r++) {
                        cp_async_16_zfill(dst + (r * 2 + 0) * 32, lane_src[r], row_bytes[r]);
                        cp_async_16_zfill(dst + (r * 2 + 1) * 32, lane_src[r] + 16, row_bytes[r]);
                    }
                } else {  // ragged last chunk: clamp the byte count per copy
#pragma unroll
                    for (int r = 0; r < R; r++)
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            long left = (n2 - (jc + 16 * h + 4 * t)) * 4;
                            uint32_t nbytes = left <= 0 ? 0u : (left < 16 ? (uint32_t)left : 16u);
                            nbytes = row_bytes[r] ? nbytes : 0u;
                            cp_async_16_zfill(dst + (r * 2 + h) * 32, nbytes ? lane_src[r] + 16 * h : Ci, nbytes);
                        }
                }
            }
#pragma unroll
            for (int r = 0; r < R; r++) lane_src[r] += chunk_step;  // this warp's next chunk (8 chunks on)
        };
        if constexpr (VEC) {
            stage = s_stage + (size_t)warp * (2 * CPL * 32);
#pragma unroll
            for (int r = 0; r < R; r++) {
                lane_src[r] = Ci + (size_t)(R * g + r) * ld + (VEC == 2 ? 8 : 4) * t + (long)warp * 32;
                row_bytes[r] = (R * g + r < E) ? 16u : 0u;
            }
            if (warp < nchunks) prefetch((long)warp * 32, 0);
            cp_async_commit();
        }

        const long trips = (nchunks + 7) / 8;
        for (long trip = 0; trip < trips; trip++) {
            const long ch = warp + 8 * trip;
            if (ch < nchunks) {
            const long j0 = ch * 32;
            float vals[R][2][4];
            if constexpr (VEC) {
                if (ch + 8 < nchunks) prefetch(j0 + 8 * 32, buf ^ 1);
                cp_async_commit();
                cp_async_wait<1>();
                __syncwarp();
                const float4 *cst = stage + buf * (CPL * 32);
                if constexpr (VEC == 2) {
#pragma unroll
                    for (int r = 0; r < R; r++) {
                        const float4 q = cst[r * 32 + lane];   // 8 fp16 values: columns 8t .. 8t+7
                        const __half2 *hq = reinterpret_cast<const __half2 *>(&q);
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const float2 lo = __half22float2(hq[2 * h]), hi = __half22float2(hq[2 * h + 1]);
                            vals[r][h][0] = lo.x, vals[r][h][1] = lo.y, vals[r][h][2] = hi.x, vals[r][h][3] = hi.y;
                        }
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < R; r++)
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            float4 q = cst[(r * 2 + h) * 32 + lane];
                            vals[r][h][0] = q.x, vals[r][h][1] = q.y, vals[r][h][2] = q.z, vals[r][h][3] = q.w;
                        }
                }
                buf ^= 1;
            } else {
                // ---- direct loads (unaligned buffers), zero outside [0,E) x [0,n2)
#pragma unroll
                for (int r = 0; r < R; r++) {
                    const int e = R * g + r;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const long col = j0 + 16 * h + 4 * t;
                        const float *src = Ci + (size_t)e * ld + col;
#pragma unroll
                        for (int u = 0; u < 4; u++) vals[r][h][u] = (e < E && col + u < n2) ? __ldg(src + u) : 0.f;
                    }
                }
            }
            if constexpr (EPS > 0) {
                // ---- Fisher-z on the epochs that belong to a complete subject
                if constexpr (FISHER) {
#pragma unroll
                    for (int r = 0; r < R; r++)
                        if (R * g + r < S_eps) {
#pragma unroll
                            for (int h = 0; h < 2; h++)
#pragma unroll
                                for (int u = 0; u < 4; u++) vals[r][h][u] = fisher_log2(vals[r][h][u]);
                        }
                }
                // ---- per (subject, column) z-score
                zscore_frag<EPS, R, 2, 4>([&](int r, int h, int u) -> float & { return vals[r][h][u]; }, g, S_eps, S_eps == E);
            }
            // ---- self-correlation column mask (optional), tf32 rounding
            if (self_col >= j0 && self_col < j0 + 32) {  // warp-uniform, one chunk per row at most
#pragma unroll
                for (int r = 0; r < R; r++)
#pragma unroll
                    for (int h = 0; h < 2; h++)
#pragma unroll
                        for (int u = 0; u < 4; u++)
                            if (j0 + (VEC == 2 ? 8 * t + 4 * h : 16 * h + 4 * t) + u == self_col) vals[r][h][u] = 0.f;
            }
            if constexpr (EPS > 0) {
                // ---- K += Z Z^T with fp16 operands (m16n8k16): z-scored values are bounded by sqrt(EPS - 1) and the
                // untouched trailing epochs hold |r| <= 1, so fp16 (11-bit significand like tf32, round to nearest
                // even) loses nothing against the tf32 path below at half the MMA instructions and one pack per two
                // values.  k-slots (2t, 2t+1) <-> columns 0, 1 and (2t+8, 2t+9) <-> columns 2, 3 of the lane's h-th
                // group of four columns, for the A and the B fragment alike.
                uint32_t hv[R][2][2];
#pragma unroll
                for (int r = 0; r < R; r++)
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        hv[r][h][0] = pack_half2_rn(vals[r][h][0], vals[r][h][1]);
                        hv[r][h][1] = pack_half2_rn(vals[r][h][2], vals[r][h][3]);
                    }
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int mu = 0; mu < MT; mu++)
#pragma unroll
                        for (int nu = 0; nu < NT; nu++)
                            mma_f16_16x8x16(acc[mu][nu], hv[2 * mu][h][0], hv[2 * mu + 1][h][0], hv[2 * mu][h][1],
                                            hv[2 * mu + 1][h][1], hv[nu][h][0], hv[nu][h][1]);
            } else {
            uint32_t tv[R][2][4];
#pragma unroll
            for (int r = 0; r < R; r++)
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int u = 0; u < 4; u++)   // round to nearest tf32 (ties away, = cvt.rna): the MMA truncates
                        tv[r][h][u] = __float_as_uint(vals[r][h][u]) + 0x1000u;
            // ---- K += Z Z^T on tensor cores.  k-step (h, w): k-slot t <-> column 2w, k-slot t+4 <-> column 2w+1 of
            // the lane's h-th group of four columns, so a B fragment is two ADJACENT registers of one 16-byte load
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int w = 0; w < 2; w++)
#pragma unroll
                    for (int mu = 0; mu < MT; mu++)
#pragma unroll
                        for (int nu = 0; nu < NT; nu++)
                            mma_tf32_16x8x8(acc[mu][nu], tv[2 * mu][h][2 * w], tv[2 * mu + 1][h][2 * w],
                                            tv[2 * mu][h][2 * w + 1], tv[2 * mu + 1][h][2 * w + 1], tv[nu][h][2 * w],
                                            tv[nu][h][2 * w + 1]);
            }
            }  // ch < nchunks
            if constexpr (R <= 4) {
                if (++since_flush == FLUSH) {
                    flush();
                    since_flush = 0;
                }
            } else {
                // R == 8: no shared memory left for per-warp partials: every FLUSH chunks a warp adds its
                // MMA accumulators into the block's s_K (fragment order: conflict-free) with shared-memory atomics
                // (round-to-nearest adds; the order in which the 8 warps arrive is not fixed, so the E > 32 kernels are
                // reproducible only to fp32 rounding, ~1e-7 relative -- the E <= 32 path above is bit-reproducible)
                if (++since_flush == FLUSH) {
                    flush_atomic();
                    since_flush = 0;
                }
            }
        }

        // ---- deterministic cross-warp reduction into s_K (epoch order restored)
        if constexpr (R <= 4) {
            flush();
            __syncthreads();
            for (int idx = threadIdx.x; idx < EP * EP; idx += 256) {
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < 8; w++) v += s_part[w * (EP * EP) + idx];
                s_K[idx] = v;
            }
            __syncthreads();
        } else {
            flush_atomic();
            __syncthreads();
        }
        // ---- write: symmetric by construction from the lower triangle (cython_blas.pyx:200-207)
        auto kval = [&](int idx) {
            const int a = idx / E, b = idx - a * E;
            if constexpr (R <= 4)
                return a >= b ? s_K[a * EP + b] : s_K[b * EP + a];
            else
                return a >= b ? s_K[frag_index(a, b)] : s_K[frag_index(b, a)];
        };
        float *Ki = K + (size_t)i * E * E;
        if (!sum_over_rows && ((E * E) & 3) == 0 && ((reinterpret_cast<uintptr_t>(Ki) & 15) == 0)) {
            // K[i] = beta * K[i] + v as 16-byte read-modify-writes with all of a thread's loads in flight at once
            // (the dependent scalar loop was latency-bound: ~16 us per row at E = 64, most of a short row's time)
            constexpr int PT = (EP * EP / 4 + 255) / 256;      // float4 pieces per thread (1 at EP = 32, 4 at EP = 64)
            float4 *K4 = reinterpret_cast<float4 *>(Ki);
            const int total4 = (E * E) >> 2;
            float4 old[PT];
#pragma unroll
            for (int u = 0; u < PT; u++) {
                const int i4 = (int)threadIdx.x + u * 256;
                old[u] = (beta != 0.f && i4 < total4) ? K4[i4] : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < PT; u++) {
                const int i4 = (int)threadIdx.x + u * 256;
                if (i4 < total4) {
                    float4 o = old[u];
                    o.x = beta * o.x + kval(4 * i4), o.y = beta * o.y + kval(4 * i4 + 1);
                    o.z = beta * o.z + kval(4 * i4 + 2), o.w = beta * o.w + kval(4 * i4 + 3);
                    K4[i4] = o;
                }
            }
        } else {
            for (int idx = threadIdx.x; idx < E * E; idx += 256) {
                const float v = kval(idx);
                if (sum_over_rows) {
                    // one kernel for all rows (Classifier): double-precision atomics when the caller gave a fp64 accumulator
                    // (50 000 row kernels of ~1e5 each: fp32 atomics would lose ~1e-5 of the sum)
                    if (K64) atomicAdd(&K64[idx], (double)v);
                    else atomicAdd(&K[idx], v);
                } else {
                    float *dst = &Ki[idx];
                    *dst = (beta == 0.f ? 0.f : beta * *dst) + v;
                }
            }
        }
        __syncthreads();
    }
}

// ============================================================================================
// Column-direction normalise + SYRK over a tiled fp32 block (symmetric pipeline, DESIGN.md 3.5):
//     K[j] += sum_{i < n} z(i, :, j) z(i, :, j)^T        for block columns j in [c0, n2)
// reads the SAME block A = [n/256][T256][E][256 i][256 j] that k_norm_syrk reads row-wise, so the GEMM does not
// have to store a transposed copy.  One CTA owns a strip of 32 adjacent columns (one 128-byte line per (epoch, row))
// and walks down the n rows 16 at a time: the brick [32 epochs][16 rows][32 columns] (64 KB) is fetched with
// cp.async into a swizzled smem buffer (double-buffered), warp w takes the 16-byte pieces of columns 4w .. 4w+3.
// Lane (g, t) holds epochs 4g .. 4g+3 x rows {2t, 2t+1, 2t+8, 2t+9} x 4 columns; the rows are the k extent of
// mma.m16n8k16 (fp16), one accumulator set per column (4 x 32 registers).  The within-subject z-score is the same
// arithmetic as in k_norm_syrk (statistics over the epochs of a subject, packed fp32x2).  Every COLS_SEG_STEPS (64) row steps the
// accumulators are folded into K through shared memory (bounds the truncating MMA accumulation chain, cf.
// k_norm_syrk) with the symmetric mirror of cython_blas.pyx:200-207.
// smem piece (line L = e*16 + row, 16-byte piece w) lives at (L*8 + (w ^ swz(L)))*16, swz(L) = ((L>>1)&3) | ((L>>6)&1)<<2:
// the cp.async writes (8 consecutive threads = one line) and the LDS.128 reads (8 lanes = 2 epochs x 4 row pairs,
// same piece w) are conflict-free.
// ============================================================================================
#ifndef FCMA_COLS_SEG_STEPS
#define FCMA_COLS_SEG_STEPS 64
#endif
constexpr int COLS_SEG_STEPS = FCMA_COLS_SEG_STEPS;   // 16-row steps between folds of the accumulators into K
constexpr int COLS_BRICKS = 3;        // 64 KB bricks in flight / in use (cp.async pipeline depth)

// One fold segment [seg0, seg1) of row steps through the cp.async brick ring: brick st+2 streams in while brick st is
// used.  prefetch(st, slot) issues this thread's copies of row step st into ring slot `slot`; step(slot) consumes the
// brick there.  Returns with every copy landed and every thread past its last read of the ring.
template <typename Prefetch, typename Step>
__device__ __forceinline__ void cols_ring_segment(long seg0, long seg1, Prefetch &&prefetch, Step &&step)
{
    static_assert(COLS_BRICKS == 3, "the ring holds the bricks st, st+1 and st+2");
    int buf = 0;
    prefetch(seg0, 0);
    cp_async_commit();
    if (seg0 + 1 < seg1) prefetch(seg0 + 1, 1);
    cp_async_commit();
    for (long st = seg0; st < seg1; st++) {
        cp_async_wait<1>();        // brick `st` has landed (this thread's copies) ...
        __syncthreads();           // ... and everybody's; every warp is also done with brick st-1,
        if (st + 2 < seg1) prefetch(st + 2, buf == 0 ? 2 : buf - 1);   // whose slot takes brick st+2
        cp_async_commit();
        step(buf);
        buf = buf == COLS_BRICKS - 1 ? 0 : buf + 1;
    }
    cp_async_wait<0>();
    __syncthreads();
}

// K += Z Z^T for one column on mma.m16n8k16 (fp16): h0[r] / h1[r] hold the z-scores of epoch slot r at k-slots
// (2t, 2t+1) / (2t+8, 2t+9); every register is both an A and a B fragment
template <int MT, int NT>
__device__ __forceinline__ void mma_zzt(float (&acc)[MT][NT][4], const uint32_t (&h0)[NT], const uint32_t (&h1)[NT])
{
#pragma unroll
    for (int mu = 0; mu < MT; mu++)
#pragma unroll
        for (int nu = 0; nu < NT; nu++)
            mma_f16_16x8x16(acc[mu][nu], h0[2 * mu], h0[2 * mu + 1], h1[2 * mu], h1[2 * mu + 1], h0[nu], h1[nu]);
}
// the same from fp32 z-scores z(r, k) of epoch slot r and row slot k (k-slots 2t, 2t+1, 2t+8, 2t+9), rounded to fp16
template <int MT, int NT, typename Z>
__device__ __forceinline__ void mma_zzt(float (&acc)[MT][NT][4], Z &&z)
{
    uint32_t h0[NT], h1[NT];
#pragma unroll
    for (int r = 0; r < NT; r++) {
        h0[r] = pack_half2_rn(z(r, 0), z(r, 1));
        h1[r] = pack_half2_rn(z(r, 2), z(r, 3));
    }
    mma_zzt(acc, h0, h1);
}

// accumulators of mma_zzt with R = NT epochs per lane -> dst [EP][EP] in (epoch, epoch) order, EP = 8R: the lane's
// rows are epochs R*g + 2mu (+1), its columns epochs R*2t + nu and R*(2t+1) + nu
template <int MT, int NT>
__device__ __forceinline__ void store_frag(float *dst, const float (&acc)[MT][NT][4], int g, int t)
{
    constexpr int R = NT, EP = 8 * R;
#pragma unroll
    for (int mu = 0; mu < MT; mu++)
#pragma unroll
        for (int nu = 0; nu < NT; nu++) {
            const int row0 = R * g + 2 * mu, row1 = row0 + 1;
            const int col0 = R * (2 * t) + nu, col1 = R * (2 * t + 1) + nu;
            dst[row0 * EP + col0] = acc[mu][nu][0];
            dst[row0 * EP + col1] = acc[mu][nu][1];
            dst[row1 * EP + col0] = acc[mu][nu][2];
            dst[row1 * EP + col1] = acc[mu][nu][3];
        }
}

// K[col] += kernel of strip column col, col < ncols, for the strip's contiguous kernels at Kst: entry (a, b) is the
// lower triangle of s_fold [col][EP*EP] mirrored (cython_blas.pyx:200-207).  The loop is latency-bound, so every thread
// keeps 8 independent loads in flight, as 16-byte read-modify-writes when E*E % 4 == 0 and Kst is 16-byte aligned.
// VEC / SCALAR: the paths a kernel compiles (only VEC: the caller guarantees the condition; only SCALAR: never vector).
template <int EP, int NTHR, bool VEC = true, bool SCALAR = true>
__device__ __forceinline__ void fold_strip(float *Kst, const float *s_fold, int E, int ncols)
{
    const int tid = threadIdx.x;
    const int EE = E * E;
    const int total = ncols * EE;
    const bool vec = VEC && (!SCALAR || ((EE & 3) == 0 && (reinterpret_cast<uintptr_t>(Kst) & 15) == 0));
    auto folded = [&](int idx) {
        const int col = idx / EE, rem = idx - col * EE;
        const int a = rem / E, b = rem - a * E;
        const float *sk = s_fold + (size_t)col * (EP * EP);
        return a >= b ? sk[a * EP + b] : sk[b * EP + a];
    };
    if (vec) {
        float4 *K4 = reinterpret_cast<float4 *>(Kst);
        const int total4 = total >> 2;
        for (int base = tid; base < total4; base += NTHR * 8) {
            float4 old[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i4 = base + u * NTHR;
                if (i4 < total4) old[u] = K4[i4];
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i4 = base + u * NTHR;
                if (i4 < total4) {
                    float4 o = old[u];
                    o.x += folded(4 * i4), o.y += folded(4 * i4 + 1), o.z += folded(4 * i4 + 2), o.w += folded(4 * i4 + 3);
                    K4[i4] = o;
                }
            }
        }
    } else {
        for (int base = tid; base < total; base += NTHR * 8) {
            float old[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i1 = base + u * NTHR;
                if (i1 < total) old[u] = Kst[i1];
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i1 = base + u * NTHR;
                if (i1 < total) Kst[i1] = old[u] + folded(i1);
            }
        }
    }
}
// CPW = columns per warp: 4 (8 warps, 4 accumulator sets, 255 registers) or 2 (16 warps, 2 accumulator sets, <= 128
// registers: twice the warps to hide the dependent statistics / shuffle chains between the block barriers)
// HALF: the block holds fp16 Fisher-z values (FCMA_FLAG_F16_INTERMEDIATE / single-product operand modes): a line
// (epoch, row) of the strip is 64 bytes, two lines share a 128-byte smem row (16-byte unit (L & 1)*4 + piece, same
// swizzle), a brick is 32 KB and warp w reads the 8 bytes of its columns 4w .. 4w+3 (LDS.64, two-way conflicts).
template <int EPS, int CPW, bool HALF>
__global__ void __launch_bounds__(32 * (32 / CPW), 1)
    k_norm_syrk_cols(const void *__restrict__ Av, long n, int E, long n2, long T256, long c0, float *K)
{
    static_assert(!HALF || CPW == 4, "the fp16 variant takes 4 columns per warp");
    constexpr int R = 4, EP = 32, MT = 2, NT = 4;
    constexpr int NTHR = 32 * (32 / CPW);      // threads per CTA
    constexpr int BRICK = HALF ? 32768 : 65536;   // bytes of one [32 epochs][16 rows][32 columns] brick
    constexpr int PPL = HALF ? 4 : 8;          // 16-byte pieces per line
    constexpr int PPT = BRICK / 16 / NTHR;     // 16-byte pieces a thread copies per brick
    constexpr int LS = NTHR / PPL;             // line stride between a thread's pieces
    using elem_t = std::conditional_t<HALF, __half, float>;
    const elem_t *A = reinterpret_cast<const elem_t *>(Av);
    extern __shared__ __align__(1024) uint8_t cs_raw[];
    uint8_t *cs = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(cs_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t brick0 = smem_u32(cs);            // 3 bricks of 64 KB; the first two double as [32 columns][EP*EP] fp32 at folds
    float *s_fold = reinterpret_cast<float *>(cs);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = (E / EPS) * EPS;
    const long nstrips = (n2 - c0 + 31) / 32;
    const long nsteps = (n + 15) / 16;

    for (long strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
        const long j0 = c0 + strip * 32;                       // first block column of the strip
        const long tjx = j0 >> 8;
        const int jo = (int)(j0 & 255);
        // issue the cp.async copies of row step `st` into brick `b`.  Thread tid copies piece w = tid & 7 of the lines
        // (tid >> 3) + 32 k, k < 16: row (tid >> 3) & 15 of epochs (tid >> 7) + 2 k -- one source offset and one
        // destination offset per thread, the rest are compile-time strides (swz of those lines = c0 | ((k >> 1) & 1) << 2)
        const int pf_w = tid & (PPL - 1), pf_line0 = tid / PPL, pf_row = pf_line0 & 15, pf_e0 = pf_line0 >> 4;
        const uint32_t pf_c = (uint32_t)((pf_line0 >> 1) & 3);
        const int pf_src = pf_e0 * 65536 + pf_row * 256 + pf_w * (HALF ? 8 : 4) + jo;
        // fp32: line L at L*128, unit = piece; fp16: lines 2m, 2m+1 share row m, unit = (L & 1)*4 + piece
        const uint32_t pf_unit = HALF ? (uint32_t)((pf_line0 & 1) * 4 + pf_w) : (uint32_t)pf_w;
        const uint32_t pf_dst = brick0 + (HALF ? (uint32_t)(pf_line0 >> 1) : (uint32_t)pf_line0) * 128u;
        auto prefetch = [&](long st, int b) {
            const long i0 = st * 16;
            const elem_t *src0 = A + ((size_t)((i0 >> 8) * T256 + tjx) * E) * 65536 + (size_t)(i0 & 255) * 256 + pf_src;
            const bool row_ok = i0 + pf_row < n;
            const uint32_t dst0 = pf_dst + (uint32_t)b * (uint32_t)BRICK;
#pragma unroll
            for (int k = 0; k < PPT; k++) {
                const bool ok = row_ok && pf_e0 + (LS / 16) * k < E;
                const uint32_t piece = (pf_unit ^ pf_c ^ (uint32_t)((((k * LS) >> 6) & 1) << 2)) << 4;
                cp_async_16_zfill_s(dst0 + (uint32_t)(k * LS) * (HALF ? 64u : 128u) + piece,
                                    ok ? src0 + (size_t)k * ((LS / 16) * 65536) : A, ok ? 16u : 0u);
            }
        };
        // this lane's reads: piece `warp` of the lines (4g + r)*16 + row(sl, t); their swizzle is t | (g & 1) << 2 for
        // every (r, sl), so one base address per thread and immediate offsets (r*16 + (sl & 1) + 8 (sl >> 1)) * 128
        const uint32_t rd_swz = (uint32_t)t | ((uint32_t)(g & 1) << 2);
        const uint32_t rd_base = HALF ? (uint32_t)(32 * g + t) * 128u + (uint32_t)(warp & 1) * 8u
                                      : (uint32_t)((R * g) * 16 + 2 * t) * 128u + ((((uint32_t)(warp * CPW) >> 2) ^ rd_swz) << 4) +
                                            (uint32_t)((warp * CPW) & 3) * 4u;
        // fp16: 16-byte unit (sl & 1)*4 + (warp >> 1), swizzled -- two variants per lane
        [[maybe_unused]] const uint32_t rd_x0 = (((uint32_t)(warp >> 1)) ^ rd_swz) << 4;
        [[maybe_unused]] const uint32_t rd_x1 = ((4u + (uint32_t)(warp >> 1)) ^ rd_swz) << 4;
        for (long seg0 = 0; seg0 < nsteps; seg0 += COLS_SEG_STEPS) {
            const long seg1 = seg0 + COLS_SEG_STEPS < nsteps ? seg0 + COLS_SEG_STEPS : nsteps;
            float acc[CPW][MT][NT][4];
#pragma unroll
            for (int c = 0; c < CPW; c++)
#pragma unroll
                for (int a = 0; a < MT; a++)
#pragma unroll
                    for (int b = 0; b < NT; b++)
#pragma unroll
                        for (int d = 0; d < 4; d++) acc[c][a][b][d] = 0.f;
            // the ring of cols_ring_segment, written out: this kernel runs at 255 registers, and with its step passed
            // as a lambda ptxas rematerialises the fp32 brick's address arithmetic differently
            static_assert(COLS_BRICKS == 3, "the ring holds the bricks st, st+1 and st+2");
            int buf = 0;
            prefetch(seg0, 0);
            cp_async_commit();
            if (seg0 + 1 < seg1) prefetch(seg0 + 1, 1);
            cp_async_commit();
            for (long st = seg0; st < seg1; st++) {
                cp_async_wait<1>();        // brick `st` has landed (this thread's copies) ...
                __syncthreads();           // ... and everybody's; every warp is also done with brick st-1,
                if (st + 2 < seg1) prefetch(st + 2, buf == 0 ? 2 : buf - 1);   // whose slot takes brick st+2
                cp_async_commit();
                // ---- this lane's 4 epochs x 4 rows x 4 columns
                float vals[R][4][CPW];
                const uint32_t bb = brick0 + (uint32_t)buf * (uint32_t)BRICK + rd_base;
#pragma unroll
                for (int r = 0; r < R; r++)
#pragma unroll
                    for (int sl = 0; sl < 4; sl++) {
                        if constexpr (HALF) {
                            const uint2 q = lds64(bb + ((sl & 1) ? rd_x1 : rd_x0) + (uint32_t)((8 * r + 4 * (sl >> 1)) * 128));
                            const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&q.x));
                            const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&q.y));
                            vals[r][sl][0] = lo.x, vals[r][sl][1] = lo.y, vals[r][sl][2] = hi.x, vals[r][sl][3] = hi.y;
                        } else if constexpr (CPW == 4) {
                            const uint4 q = lds128(bb + (uint32_t)((r * 16 + (sl & 1) + 8 * (sl >> 1)) * 128));
                            vals[r][sl][0] = __uint_as_float(q.x), vals[r][sl][1] = __uint_as_float(q.y);
                            vals[r][sl][2] = __uint_as_float(q.z), vals[r][sl][3] = __uint_as_float(q.w);
                        } else {
                            const uint2 q = lds64(bb + (uint32_t)((r * 16 + (sl & 1) + 8 * (sl >> 1)) * 128));
                            vals[r][sl][0] = __uint_as_float(q.x), vals[r][sl][1] = __uint_as_float(q.y);
                        }
                    }
                // ---- within-subject z-score per (row, column), then K_j += Z Z^T per column
                zscore_frag<EPS, R, 4, CPW>([&](int r, int sl, int u) -> float & { return vals[r][sl][u]; }, g, S_eps);
#pragma unroll
                for (int c = 0; c < CPW; c++) mma_zzt(acc[c], [&](int r, int sl) { return vals[r][sl][c]; });
                buf = buf == COLS_BRICKS - 1 ? 0 : buf + 1;
            }
            cp_async_wait<0>();
            __syncthreads();
            // ---- fold the accumulators into K: registers -> smem [32 columns][EP*EP] -> mirrored, coalesced += on K
#pragma unroll
            for (int c = 0; c < CPW; c++) store_frag(s_fold + (size_t)(warp * CPW + c) * (EP * EP), acc[c], g, t);
            __syncthreads();
            const long ncols = n2 - j0 < 32 ? n2 - j0 : 32;       // real columns of this strip
            fold_strip<EP, NTHR>(K + (size_t)j0 * (E * E), s_fold, E, (int)ncols);   // the strip's kernels are contiguous
            __syncthreads();
        }
    }
}

// ============================================================================================
// Column-direction pass, version 2 (FCMA_FLAG_COLS_V2, fp32 block): normalise ONCE per value in a thread-per-row layout,
// then feed the MMAs with ldmatrix.  An opt-in alternative to k_norm_syrk_cols with the same results.
//
// k_norm_syrk_cols above loads a brick straight into mma fragment layout (lane = (4 epochs, 4 rows)), so the statistics
// of a subject are spread over lanes (shuffles), every value pair has to be re-paired for the packed fp32x2 FMAs
// (15 % of its dynamic instructions are IMAD.MOV) and each lane repeats its partner's subject_coeffs: ~680 warp
// instructions per warp and brick at two warps per scheduler.
// Here warp w still owns columns 4w .. 4w+3 of the 32-column strip, but per brick [32 epochs][16 rows][32 columns]
//   phase 1: lane l takes row (l & 15) and epochs 16*(l >> 4) .. +15: sixteen LDS.128 (4 adjacent columns of one
//            (epoch, row) each), the subject statistics are plain in-thread sums over epochs on NATURAL fp32x2 pairs
//            (columns 0|1 and 2|3) -- no shuffles (EPS = 32: one exchange with lane l ^ 16), one subject_coeffs per (subject,
//            column pair); the z-scored values are rounded to fp16 and stored as [column][row][32 epochs] (64 B per
//            (column, row), 16-byte pieces swizzled with (row >> 1) & 3, bit 2 of the bank group from row & 1) into the
//            warp's own 4 KB staging buffer;
//   phase 2: per column two ldmatrix.x4.trans (rows 0-7 -> k-slots 2t, 2t+1; rows 8-15 -> k-slots 2t+8, 2t+9) deliver
//            the eight fragment registers that serve as A AND B operands of the eight mma.m16n8k16 of Z Z^T, with lane
//            g <-> epoch 8*block + g: the accumulators are in NATURAL epoch order (no permutation to undo).
// Only a __syncwarp separates the phases (a warp consumes what it staged).  The cp.async brick ring, the folds and the
// arithmetic are shared with k_norm_syrk_cols (cols_ring_segment, subject_coeffs, mma_zzt; the fold is fold_strip's, written
// out); the smem line swizzle is L & 7 (phase 1 reads 8 consecutive rows of one epoch).
// ============================================================================================
// CPW = 4: 8 warps x 4 columns (255 registers); CPW = 2: 16 warps x 2 columns (<= 128 registers, LDS.64): four warps per
// scheduler instead of two
template <int EPS, int CPW>
__global__ void __launch_bounds__(32 * (32 / CPW), 1)
    k_norm_syrk_cols2(const float *__restrict__ A, long n, int E, long n2, long T256, long c0, float *K)
{
    constexpr int EP = 32, MT = 2, NT = 4, NTHR = 32 * (32 / CPW);
    constexpr int BRICK = 65536, PPT = BRICK / 16 / NTHR, LS = NTHR / 8;     // pieces per thread, lines between them
    constexpr uint32_t STAGE_OFF = COLS_BRICKS * BRICK;                      // 8 x 4 KB fp16 staging buffers behind the bricks
    extern __shared__ __align__(1024) uint8_t cs_raw[];
    uint8_t *cs = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(cs_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t brick0 = smem_u32(cs);
    float *s_fold = reinterpret_cast<float *>(cs);         // [32 columns][EP*EP] fp32 (128 KB) overlays bricks 0 and 1 at folds
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = (E / EPS) * EPS;
    const long nstrips = (n2 - c0 + 31) / 32;
    const long nsteps = (n + 15) / 16;
    // phase 1: this lane's row and epoch half
    const int prow = lane & 15, phalf = lane >> 4;
    const uint32_t rd_piece = CPW == 4 ? (uint32_t)warp : (uint32_t)warp >> 1;
    const uint32_t rd_base = (uint32_t)((phalf * 16) * 16 + prow) * 128u + ((rd_piece ^ ((uint32_t)prow & 7u)) << 4) +
                             (CPW == 4 ? 0u : ((uint32_t)warp & 1u) * 8u);
    const uint32_t stage = brick0 + STAGE_OFF + (uint32_t)warp * (uint32_t)(CPW * 1024);
    // staged piece (column c, row, epoch block eb) lives at  c*1024 + row*64 + ((eb ^ ((row >> 1) & 3)) << 4)
    const uint32_t st_row = stage + (uint32_t)prow * 64u;
    const uint32_t st_swz = ((uint32_t)prow >> 1) & 3u;
    // phase 2: ldmatrix row address of this lane: matrix (lane >> 3) = epoch block, row (lane & 7) (+8 for the second load)
    const uint32_t lm_row = (uint32_t)lane & 7u, lm_eb = (uint32_t)lane >> 3;
    const uint32_t lm_lo = stage + lm_row * 64u + ((lm_eb ^ ((lm_row >> 1) & 3u)) << 4);
    const uint32_t lm_hi = stage + (lm_row + 8u) * 64u + ((lm_eb ^ (((lm_row + 8u) >> 1) & 3u)) << 4);

    for (long strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
        const long j0 = c0 + strip * 32;
        const long tjx = j0 >> 8;
        const int jo = (int)(j0 & 255);
        // cp.async: thread tid copies piece w = tid & 7 of the lines (tid >> 3) + 32 k, k < 16 (row (tid >> 3) & 15 of
        // epochs (tid >> 7) + 2 k); L & 7 is the same for all of them
        const int pf_w = tid & 7, pf_line0 = tid >> 3, pf_row = pf_line0 & 15, pf_e0 = pf_line0 >> 4;
        const int pf_src = pf_e0 * 65536 + pf_row * 256 + pf_w * 4 + jo;
        constexpr int EPK = LS / 16;          // epochs between a thread's pieces
        const uint32_t pf_dst = brick0 + (uint32_t)pf_line0 * 128u + ((((uint32_t)pf_w) ^ ((uint32_t)pf_line0 & 7u)) << 4);
        auto prefetch = [&](long st, int b) {
            const long i0 = st * 16;
            const float *src0 = A + ((size_t)((i0 >> 8) * T256 + tjx) * E) * 65536 + (size_t)(i0 & 255) * 256 + pf_src;
            const bool row_ok = i0 + pf_row < n;
            const uint32_t dst0 = pf_dst + (uint32_t)b * (uint32_t)BRICK;
#pragma unroll
            for (int k = 0; k < PPT; k++) {
                const bool ok = row_ok && pf_e0 + EPK * k < E;
                cp_async_16_zfill_s(dst0 + (uint32_t)(k * LS) * 128u, ok ? src0 + (size_t)k * (EPK * 65536) : A, ok ? 16u : 0u);
            }
        };
        for (long seg0 = 0; seg0 < nsteps; seg0 += COLS_SEG_STEPS) {
            const long seg1 = seg0 + COLS_SEG_STEPS < nsteps ? seg0 + COLS_SEG_STEPS : nsteps;
            float acc[CPW][MT][NT][4];
#pragma unroll
            for (int c = 0; c < CPW; c++)
#pragma unroll
                for (int a = 0; a < MT; a++)
#pragma unroll
                    for (int b = 0; b < NT; b++)
#pragma unroll
                        for (int d = 0; d < 4; d++) acc[c][a][b][d] = 0.f;
            cols_ring_segment(seg0, seg1, prefetch, [&](int buf) {
                const uint32_t bb = brick0 + (uint32_t)buf * (uint32_t)BRICK + rd_base;
                // ---- phase 1: 16 epochs x 4 columns of this lane's row, 8 epochs (one staged piece) at a time
                float2 lo[16], hi[CPW == 4 ? 16 : 1];     // columns (0, 1) and (2, 3) of epoch 16*phalf + e
#pragma unroll
                for (int e = 0; e < 16; e++) {
                    if constexpr (CPW == 4) {
                        const uint4 q = lds128(bb + (uint32_t)e * 2048u);
                        lo[e] = make_float2(__uint_as_float(q.x), __uint_as_float(q.y));
                        hi[e] = make_float2(__uint_as_float(q.z), __uint_as_float(q.w));
                    } else {
                        const uint2 q = lds64(bb + (uint32_t)e * 2048u);
                        lo[e] = make_float2(__uint_as_float(q.x), __uint_as_float(q.y));
                    }
                }
                constexpr int SPAN = EPS < 16 ? EPS : 16;          // epochs of one subject inside this lane
#pragma unroll
                for (int s0 = 0; s0 < 16; s0 += SPAN) {
                    float2 ml = splat2(0.f), mh = splat2(0.f), ql = splat2(0.f), qh = splat2(0.f);
#pragma unroll
                    for (int e = s0; e < s0 + SPAN; e++) {
                        ml = fadd2(ml, lo[e]), ql = ffma2(lo[e], lo[e], ql);
                        if constexpr (CPW == 4) mh = fadd2(mh, hi[e]), qh = ffma2(hi[e], hi[e], qh);
                    }
                    if constexpr (EPS == 32) {       // the subject's other 16 epochs live in lane ^ 16
                        ml.x += __shfl_xor_sync(0xffffffffu, ml.x, 16), ml.y += __shfl_xor_sync(0xffffffffu, ml.y, 16);
                        ql.x += __shfl_xor_sync(0xffffffffu, ql.x, 16), ql.y += __shfl_xor_sync(0xffffffffu, ql.y, 16);
                        if constexpr (CPW == 4) {
                            mh.x += __shfl_xor_sync(0xffffffffu, mh.x, 16), mh.y += __shfl_xor_sync(0xffffffffu, mh.y, 16);
                            qh.x += __shfl_xor_sync(0xffffffffu, qh.x, 16), qh.y += __shfl_xor_sync(0xffffffffu, qh.y, 16);
                        }
                    }
                    float2 il, cl, ih = splat2(0.f), ch = splat2(0.f);
                    subject_coeffs<EPS>(ml, ql, il, cl);
                    if constexpr (CPW == 4) subject_coeffs<EPS>(mh, qh, ih, ch);
                    if (16 * phalf + s0 < S_eps) {       // epochs outside a complete subject stay as they are
#pragma unroll
                        for (int e = s0; e < s0 + SPAN; e++) {
                            lo[e] = ffma2(lo[e], il, cl);
                            if constexpr (CPW == 4) hi[e] = ffma2(hi[e], ih, ch);
                        }
                    }
                }
                // ---- stage: per column two 16-byte pieces (epochs 16*phalf .. +7 and +8 .. +15) of this lane's row
#pragma unroll
                for (int pc = 0; pc < 2; pc++) {
                    const uint32_t piece = st_row + ((((uint32_t)(2 * phalf + pc)) ^ st_swz) << 4);
                    const int e0 = 8 * pc;
                    sts128(piece + 0 * 1024u, pack_half2_rn(lo[e0].x, lo[e0 + 1].x), pack_half2_rn(lo[e0 + 2].x, lo[e0 + 3].x),
                           pack_half2_rn(lo[e0 + 4].x, lo[e0 + 5].x), pack_half2_rn(lo[e0 + 6].x, lo[e0 + 7].x));
                    sts128(piece + 1 * 1024u, pack_half2_rn(lo[e0].y, lo[e0 + 1].y), pack_half2_rn(lo[e0 + 2].y, lo[e0 + 3].y),
                           pack_half2_rn(lo[e0 + 4].y, lo[e0 + 5].y), pack_half2_rn(lo[e0 + 6].y, lo[e0 + 7].y));
                    if constexpr (CPW == 4) {
                        sts128(piece + 2 * 1024u, pack_half2_rn(hi[e0].x, hi[e0 + 1].x), pack_half2_rn(hi[e0 + 2].x, hi[e0 + 3].x),
                               pack_half2_rn(hi[e0 + 4].x, hi[e0 + 5].x), pack_half2_rn(hi[e0 + 6].x, hi[e0 + 7].x));
                        sts128(piece + 3 * 1024u, pack_half2_rn(hi[e0].y, hi[e0 + 1].y), pack_half2_rn(hi[e0 + 2].y, hi[e0 + 3].y),
                               pack_half2_rn(hi[e0 + 4].y, hi[e0 + 5].y), pack_half2_rn(hi[e0 + 6].y, hi[e0 + 7].y));
                    }
                }
                __syncwarp();
                // ---- phase 2: K_j += Z Z^T for the warp's four columns
#pragma unroll
                for (int c = 0; c < CPW; c++) {
                    uint32_t h0[4], h1[4];      // epoch block r: rows (2t, 2t+1) / (2t+8, 2t+9) of epoch 8r + g
                    ldmatrix_x4_trans(lm_lo + (uint32_t)c * 1024u, h0[0], h0[1], h0[2], h0[3]);
                    ldmatrix_x4_trans(lm_hi + (uint32_t)c * 1024u, h1[0], h1[1], h1[2], h1[3]);
                    mma_zzt(acc[c], h0, h1);
                }
                __syncwarp();      // the staging buffer is rewritten in the next step
            });
            // ---- fold the accumulators into K: registers -> smem [32 columns][EP*EP] -> mirrored, coalesced += on K.
            // Natural epoch order: acc[c][mu][nu][{0,1}] = K[16 mu + g][8 nu + 2t + {0,1}], [{2,3}] = row 16 mu + g + 8.
#pragma unroll
            for (int c = 0; c < CPW; c++) {
                float *dstk = s_fold + (size_t)(warp * CPW + c) * (EP * EP);
#pragma unroll
                for (int mu = 0; mu < MT; mu++)
#pragma unroll
                    for (int nu = 0; nu < NT; nu++) {
                        const int row0 = 16 * mu + g, col0 = 8 * nu + 2 * t;
                        *reinterpret_cast<float2 *>(&dstk[row0 * EP + col0]) = make_float2(acc[c][mu][nu][0], acc[c][mu][nu][1]);
                        *reinterpret_cast<float2 *>(&dstk[(row0 + 8) * EP + col0]) = make_float2(acc[c][mu][nu][2], acc[c][mu][nu][3]);
                    }
            }
            __syncthreads();
            const int EE = E * E;
            const long ncols = n2 - j0 < 32 ? n2 - j0 : 32;       // real columns of this strip
            const int total = (int)ncols * EE;
            float *Kst = K + (size_t)j0 * EE;                     // the strip's kernels are contiguous
            auto folded = [&](int idx) {
                const int col = idx / EE, rem = idx - col * EE;
                const int a = rem / E, b = rem - a * E;
                const float *sk = s_fold + (size_t)col * (EP * EP);
                return a >= b ? sk[a * EP + b] : sk[b * EP + a];
            };
            // fold_strip, written out: at 16 warps x 128 registers (CPW = 2), calling the helper lets the compiler hoist
            // the brick copies' address arithmetic out of the strip loop, which adds spills (52 -> 148 bytes of stores at
            // EPS = 1) and ran 2.6 % slower (H100 80GB HBM3, 700 W limit)
            if ((EE & 3) == 0 && ((reinterpret_cast<uintptr_t>(Kst) & 15) == 0)) {
                float4 *K4 = reinterpret_cast<float4 *>(Kst);
                const int total4 = total >> 2;
                for (int base = tid; base < total4; base += NTHR * 8) {
                    float4 old[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i4 = base + u * NTHR;
                        if (i4 < total4) old[u] = K4[i4];
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i4 = base + u * NTHR;
                        if (i4 < total4) {
                            float4 o = old[u];
                            o.x += folded(4 * i4), o.y += folded(4 * i4 + 1), o.z += folded(4 * i4 + 2), o.w += folded(4 * i4 + 3);
                            K4[i4] = o;
                        }
                    }
                }
            } else {
                for (int base = tid; base < total; base += NTHR * 8) {
                    float old[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i1 = base + u * NTHR;
                        if (i1 < total) old[u] = Kst[i1];
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i1 = base + u * NTHR;
                        if (i1 < total) Kst[i1] = old[u] + folded(i1);
                    }
                }
            }
            __syncthreads();
        }
    }
}

// ============================================================================================
// Column-direction pass for E <= 16 (default there, fp32 block): the structure of version 2 with 16-epoch bricks
// [16 epochs][16 rows][32 columns] (32 KB) instead of bricks padded to 32 epochs -- half the shared-memory traffic,
// statistics and MMAs per byte of the block (BASELINE configs[1], E = 16: the padded kernels ran at 0.40 of the HBM peak).
//   phase 1: lane l takes row (l & 15), ALL 16 epochs and two of the warp's four columns (l >> 4): sixteen LDS.64, in-thread
//            subject statistics on one natural fp32x2 pair, z-scores staged as fp16 [column][row][16 epochs] (32 B per
//            (column, row); the two 16-byte pieces swapped for rows 4-7 / 12-15 so that eight rows hit eight bank groups);
//   phase 2: per column ONE ldmatrix.x4.trans = {epochs 0-7, 8-15} x {rows 0-7, 8-15} -> the four fragment registers of
//            the two mma.m16n8k16 of a 16 x 16 kernel; 8 accumulator registers per column.
// 3 bricks + 16 KB of staging = 112 KB and ~110 registers: two CTAs per SM.
// ============================================================================================
template <int EPS>
__global__ void __launch_bounds__(256, 2)
    k_norm_syrk_cols16(const float *__restrict__ A, long n, int E, long n2, long T256, long c0, float *K)
{
    static_assert(EPS <= 16, "a subject spans at most the 16 epochs of this kernel");
    constexpr int EP = 16, NT = 2, CPW = 4, NTHR = 256;
    constexpr int BRICK = 32768, PPT = BRICK / 16 / NTHR, LS = NTHR / 8;     // 8 pieces per thread, 32 lines apart
    constexpr uint32_t STAGE_OFF = COLS_BRICKS * BRICK;
    extern __shared__ __align__(1024) uint8_t cs_raw[];
    // 128-byte alignment is all the swizzles need; the smaller slack keeps two CTAs (2 x 113 KB) inside one SM's 228 KB
    uint8_t *cs = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(cs_raw) + 127) & ~uintptr_t(127));
    const uint32_t brick0 = smem_u32(cs);
    float *s_fold = reinterpret_cast<float *>(cs);         // [32 columns][EP*EP] fp32 (32 KB) overlays brick 0 at folds
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = (E / EPS) * EPS;
    const long nstrips = (n2 - c0 + 31) / 32;
    const long nsteps = (n + 15) / 16;
    const int prow = lane & 15, pcp = lane >> 4;           // phase 1: row, column pair (columns 2*pcp, 2*pcp + 1 of the warp's 4)
    const uint32_t rd_base = (uint32_t)prow * 128u + ((((uint32_t)warp) ^ ((uint32_t)prow & 7u)) << 4) + (uint32_t)pcp * 8u;
    const uint32_t stage = brick0 + STAGE_OFF + (uint32_t)warp * 2048u;
    // staged piece (column c, row, epoch block eb in {0, 1}) at  c*512 + row*32 + ((eb ^ ((row >> 2) & 1)) << 4)
    const uint32_t st_row = stage + (uint32_t)prow * 32u;
    const uint32_t st_swz = ((uint32_t)prow >> 2) & 1u;
    // ldmatrix: matrix m = lane >> 3: epoch block m & 1, rows 8*(m >> 1) .. +7; this lane supplies row (lane & 7) of it
    const uint32_t lm_r = ((uint32_t)lane & 7u) + 8u * ((uint32_t)lane >> 4), lm_eb = ((uint32_t)lane >> 3) & 1u;
    const uint32_t lm_addr = stage + lm_r * 32u + ((lm_eb ^ ((lm_r >> 2) & 1u)) << 4);

    for (long strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
        const long j0 = c0 + strip * 32;
        const long tjx = j0 >> 8;
        const int jo = (int)(j0 & 255);
        const int pf_w = tid & 7, pf_line0 = tid >> 3, pf_row = pf_line0 & 15, pf_e0 = pf_line0 >> 4;
        const int pf_src = pf_e0 * 65536 + pf_row * 256 + pf_w * 4 + jo;
        const uint32_t pf_dst = brick0 + (uint32_t)pf_line0 * 128u + ((((uint32_t)pf_w) ^ ((uint32_t)pf_line0 & 7u)) << 4);
        auto prefetch = [&](long st, int b) {
            const long i0 = st * 16;
            const float *src0 = A + ((size_t)((i0 >> 8) * T256 + tjx) * E) * 65536 + (size_t)(i0 & 255) * 256 + pf_src;
            const bool row_ok = i0 + pf_row < n;
            const uint32_t dst0 = pf_dst + (uint32_t)b * (uint32_t)BRICK;
#pragma unroll
            for (int k = 0; k < PPT; k++) {
                const bool ok = row_ok && pf_e0 + 2 * k < E;
                cp_async_16_zfill_s(dst0 + (uint32_t)(k * LS) * 128u, ok ? src0 + (size_t)k * (2 * 65536) : A, ok ? 16u : 0u);
            }
        };
        for (long seg0 = 0; seg0 < nsteps; seg0 += COLS_SEG_STEPS) {
            const long seg1 = seg0 + COLS_SEG_STEPS < nsteps ? seg0 + COLS_SEG_STEPS : nsteps;
            float acc[CPW][NT][4];
#pragma unroll
            for (int c = 0; c < CPW; c++)
#pragma unroll
                for (int b = 0; b < NT; b++)
#pragma unroll
                    for (int d = 0; d < 4; d++) acc[c][b][d] = 0.f;
            cols_ring_segment(seg0, seg1, prefetch, [&](int buf) {
                const uint32_t bb = brick0 + (uint32_t)buf * (uint32_t)BRICK + rd_base;
                // ---- phase 1: 16 epochs x 2 columns of this lane's row
                float2 v[16];
#pragma unroll
                for (int e = 0; e < 16; e++) {
                    const uint2 q = lds64(bb + (uint32_t)e * 2048u);
                    v[e] = make_float2(__uint_as_float(q.x), __uint_as_float(q.y));
                }
#pragma unroll
                for (int s0 = 0; s0 < 16; s0 += EPS) {
                    float2 m = splat2(0.f), q2 = splat2(0.f);
#pragma unroll
                    for (int e = s0; e < s0 + EPS; e++) m = fadd2(m, v[e]), q2 = ffma2(v[e], v[e], q2);
                    float2 inv, mi;
                    subject_coeffs<EPS>(m, q2, inv, mi);
                    if (s0 < S_eps) {
#pragma unroll
                        for (int e = s0; e < s0 + EPS; e++) v[e] = ffma2(v[e], inv, mi);
                    }
                }
                // ---- stage: per column two 16-byte pieces (epochs 0-7 and 8-15) of this lane's row
#pragma unroll
                for (int pc = 0; pc < 2; pc++) {
                    const uint32_t piece = st_row + ((((uint32_t)pc) ^ st_swz) << 4) + (uint32_t)(2 * pcp) * 512u;
                    const int e0 = 8 * pc;
                    sts128(piece, pack_half2_rn(v[e0].x, v[e0 + 1].x), pack_half2_rn(v[e0 + 2].x, v[e0 + 3].x),
                           pack_half2_rn(v[e0 + 4].x, v[e0 + 5].x), pack_half2_rn(v[e0 + 6].x, v[e0 + 7].x));
                    sts128(piece + 512u, pack_half2_rn(v[e0].y, v[e0 + 1].y), pack_half2_rn(v[e0 + 2].y, v[e0 + 3].y),
                           pack_half2_rn(v[e0 + 4].y, v[e0 + 5].y), pack_half2_rn(v[e0 + 6].y, v[e0 + 7].y));
                }
                __syncwarp();
                // ---- phase 2: one ldmatrix and two MMAs per column
#pragma unroll
                for (int c = 0; c < CPW; c++) {
                    uint32_t h00, h01, h10, h11;    // h{rows half}{epoch block}: epochs 8*block + g, rows (2t, 2t+1) (+8)
                    ldmatrix_x4_trans(lm_addr + (uint32_t)c * 512u, h00, h01, h10, h11);
#pragma unroll
                    for (int nu = 0; nu < NT; nu++)
                        mma_f16_16x8x16(acc[c][nu], h00, h01, h10, h11, nu == 0 ? h00 : h01, nu == 0 ? h10 : h11);
                }
                __syncwarp();
            });
            // ---- fold: acc[c][nu][{0,1}] = K[g][8 nu + 2t + {0,1}], [{2,3}] = row g + 8
#pragma unroll
            for (int c = 0; c < CPW; c++) {
                float *dstk = s_fold + (size_t)(warp * CPW + c) * (EP * EP);
#pragma unroll
                for (int nu = 0; nu < NT; nu++) {
                    const int col0 = 8 * nu + 2 * t;
                    *reinterpret_cast<float2 *>(&dstk[g * EP + col0]) = make_float2(acc[c][nu][0], acc[c][nu][1]);
                    *reinterpret_cast<float2 *>(&dstk[(g + 8) * EP + col0]) = make_float2(acc[c][nu][2], acc[c][nu][3]);
                }
            }
            __syncthreads();
            const long ncols = n2 - j0 < 32 ? n2 - j0 : 32;
            fold_strip<EP, NTHR, false>(K + (size_t)j0 * (E * E), s_fold, E, (int)ncols);
            __syncthreads();
        }
    }
}

// ============================================================================================
// Column-direction pass for 32 < E <= 64 (fp32 block): the 64 x 64 accumulator of ONE column voxel fills a warp's registers
// (4 x 8 MMA tiles = 128), so a CTA of 8 warps owns a strip of 8 adjacent columns -- 32 bytes of every (epoch, row) line; the
// CTAs of neighbouring strips walk down the same rows at the same time and find the rest of the 128-byte line in L2.  A brick
// is [64 epochs][16 rows][8 columns] = 32 KB; 4-byte cp.async scatter it into a column-major shared layout
//     word(col, e, row) = col * 1092 + (e >> 3) * 136 + (e & 7) * 16 + row
// (136: the eight epoch groups of a half warp's LDS.64 fall into distinct banks; 1092: the eight columns of a copying warp do),
// so lane (g, t) of warp `col` reads its 8 epochs 8g .. 8g+7 x rows {2t, 2t+1}, {2t+8, 2t+9} with 16 conflict-free LDS.64.
// Statistics, z-score, fragment roles and the fold are k_norm_syrk_cols's shared helpers (zscore_frag, mma_zzt, store_frag,
// fold_strip) with R = 8 epochs per lane.
// ============================================================================================
template <int EPS>
__global__ void __launch_bounds__(256, 1)
    k_norm_syrk_cols64(const float *__restrict__ A, long n, int E, long n2, long T256, long c0, float *K)
{
    constexpr int R = 8, EP = 64, MT = 4, NT = 8, NTHR = 256;
    constexpr int COLW = 1092;                 // words per column of a brick
    constexpr int BRICK = 8 * COLW * 4;        // bytes
    extern __shared__ __align__(1024) uint8_t cs_raw[];
    uint8_t *cs = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(cs_raw) + 127) & ~uintptr_t(127));
    const uint32_t brick0 = smem_u32(cs);            // 3 bricks; the fold area [8 columns][64*64] fp32 (128 KB) overlays them
    float *s_fold = reinterpret_cast<float *>(cs);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = (E / EPS) * EPS;
    const long nstrips = (n2 - c0 + 7) / 8;
    const long nsteps = (n + 15) / 16;
    // copies: thread = (column tid & 7, row (tid >> 3) & 15, epochs (tid >> 7) + 2k, k < 32)
    const int pf_col = tid & 7, pf_row = (tid >> 3) & 15, pf_e0 = tid >> 7;
    const uint32_t pf_dst = brick0 + (uint32_t)(pf_col * COLW + pf_e0 * 16 + pf_row) * 4u;
    const uint32_t rd_base = (uint32_t)(warp * COLW + g * 136 + 2 * t) * 4u;

    for (long strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
        const long j0 = c0 + strip * 8;
        const long tjx = j0 >> 8;
        const int jo = (int)(j0 & 255);
        const bool col_ok = j0 + pf_col < n2;
        const bool strip_full = E == 64 && j0 + 8 <= n2;
        auto prefetch = [&](long st, int b) {
            const long i0 = st * 16;
            const float *src0 = A + ((size_t)((i0 >> 8) * T256 + tjx) * E) * 65536 + (size_t)((i0 & 255) + pf_row) * 256 + jo + pf_col +
                                (size_t)pf_e0 * 65536;
            const uint32_t dst0 = pf_dst + (uint32_t)b * (uint32_t)BRICK;
            if (strip_full && i0 + 16 <= n) {
                // the common case (CTA-uniform): 32 unconditional copies off one source and one destination register
#pragma unroll
                for (int k = 0; k < 32; k++)
                    cp_async_4_s(dst0 + (uint32_t)((k >> 2) * 136 + 2 * (k & 3) * 16) * 4u, src0 + (size_t)k * 131072);
                return;
            }
            const bool ok0 = col_ok && i0 + pf_row < n;
#pragma unroll 4
            for (int k = 0; k < 32; k++) {
                const bool ok = ok0 && pf_e0 + 2 * k < E;
                // epoch e = pf_e0 + 2k: group k >> 2, slot pf_e0 + 2 (k & 3)
                cp_async_4_zfill_s(dst0 + (uint32_t)((k >> 2) * 136 + 2 * (k & 3) * 16) * 4u, ok ? src0 + (size_t)k * 131072 : A,
                                   ok ? 4u : 0u);
            }
        };
        for (long seg0 = 0; seg0 < nsteps; seg0 += COLS_SEG_STEPS) {
            const long seg1 = seg0 + COLS_SEG_STEPS < nsteps ? seg0 + COLS_SEG_STEPS : nsteps;
            float acc[MT][NT][4];
#pragma unroll
            for (int a = 0; a < MT; a++)
#pragma unroll
                for (int b = 0; b < NT; b++)
#pragma unroll
                    for (int d = 0; d < 4; d++) acc[a][b][d] = 0.f;
            cols_ring_segment(seg0, seg1, prefetch, [&](int buf) {
                float2 lo[R], hi[R];     // rows (2t, 2t+1) and (2t+8, 2t+9) of epoch 8g + r, this warp's column
                const uint32_t bb = brick0 + (uint32_t)buf * (uint32_t)BRICK + rd_base;
#pragma unroll
                for (int r = 0; r < R; r++) {
                    const uint2 q0 = lds64(bb + (uint32_t)(r * 16) * 4u);
                    const uint2 q1 = lds64(bb + (uint32_t)(r * 16 + 8) * 4u);
                    lo[r] = make_float2(__uint_as_float(q0.x), __uint_as_float(q0.y));
                    hi[r] = make_float2(__uint_as_float(q1.x), __uint_as_float(q1.y));
                }
                // z-score: two row slots (the pair) per packed op, one column
                zscore_frag<EPS, R, 1, 2>([&](int r, int, int u) -> float & { return u ? lo[r].y : lo[r].x; }, g, S_eps);
                zscore_frag<EPS, R, 1, 2>([&](int r, int, int u) -> float & { return u ? hi[r].y : hi[r].x; }, g, S_eps);
                mma_zzt(acc, [&](int r, int sl) {
                    const float2 p = sl < 2 ? lo[r] : hi[r];
                    return sl & 1 ? p.y : p.x;
                });
            });
            // ---- fold: registers -> smem [8 columns][64*64] -> mirrored, coalesced += on K
            store_frag(s_fold + (size_t)warp * (EP * EP), acc, g, t);
            __syncthreads();
            const int EE = E * E;
            const long ncols = n2 - j0 < 8 ? n2 - j0 : 8;
            const int total = (int)ncols * EE;
            float *Kst = K + (size_t)j0 * EE;
            if (E == 64 && ((reinterpret_cast<uintptr_t>(Kst) & 15) == 0)) {
                // 16-byte read-modify-write, 8 independent loads in flight per thread; entry (a, b) of column `col`
                float4 *K4 = reinterpret_cast<float4 *>(Kst);
                const int total4 = total >> 2;
                auto folded4 = [&](int i4) {
                    const int col = i4 >> 10, a = (i4 >> 4) & 63, b = (i4 & 15) * 4;
                    const float *sk = s_fold + (size_t)col * (EP * EP);
                    float4 r;
                    r.x = a >= b ? sk[a * EP + b] : sk[b * EP + a];
                    r.y = a >= b + 1 ? sk[a * EP + b + 1] : sk[(b + 1) * EP + a];
                    r.z = a >= b + 2 ? sk[a * EP + b + 2] : sk[(b + 2) * EP + a];
                    r.w = a >= b + 3 ? sk[a * EP + b + 3] : sk[(b + 3) * EP + a];
                    return r;
                };
                for (int base = tid; base < total4; base += NTHR * 8) {
                    float4 old[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i4 = base + u * NTHR;
                        if (i4 < total4) old[u] = K4[i4];
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const int i4 = base + u * NTHR;
                        if (i4 < total4) {
                            const float4 f = folded4(i4);
                            float4 o = old[u];
                            o.x += f.x, o.y += f.y, o.z += f.z, o.w += f.w;
                            K4[i4] = o;
                        }
                    }
                }
            } else {
                fold_strip<EP, NTHR, false>(Kst, s_fold, E, (int)ncols);
            }
            __syncthreads();
        }
    }
}

// ============================================================================================
// Column-direction pass, TMA version (FCMA_FLAG_COLS_TMA, needs E % 4 == 0): same arithmetic as k_norm_syrk_cols, but
//   * a brick [32 epochs][16 rows][32 columns] arrives through ONE 5-D bulk tensor copy (UTMALDG) issued by one elected
//     lane -- the 4096 LDGSTS per brick (8 LSU cycles each, the same port the LDS reads need) and their address
//     arithmetic are gone;
//   * bricks live in a 3-slot ring guarded by full/empty mbarriers: a warp waits for ITS brick and releases it when
//     it is done, so warps run up to a brick apart instead of meeting at a bar.sync every 64 KB.
// The tiled block [tile group][E][256 i][256 j] is described to TMA as a 5-D tensor whose dimension ORDER is chosen
// for the reader, not for memory:   (j, i%4, tile group * E/4 + e/4, (i%256)/4, e%4)   with box (32, 4, 8, 4, 4).
// Shared-memory line L = i%4 + 4*(e/4) + 32*(i/4 %4) + 128*(e%4) then lands at L*128 with the hardware 128-byte
// swizzle (16-byte piece ^ (L & 7)).  Lane (g, t) of the mma fragment layout takes epochs 4g .. 4g+3 and rows
// {t, t+4, t+8, t+12} (which rows a k-slot stands for is irrelevant to a sum over rows, as long as every lane uses the
// same mapping), so the eight lanes of an LDS.128 phase (g in {2h, 2h+1}, t in 0..3) read lines with eight different
// L & 7 = t + 4 (g & 1): conflict-free without a custom swizzle.  Offsets of (epoch r, row slot sl) are multiples of
// 4 KB: immediate operands.  Rows >= n of a ragged last row tile hold stale scratch: masked after the load.
// Epochs [E, 32) of the box belong to the next tile group (or are zero-filled beyond the tensor): they only reach
// accumulator rows / columns >= E, which are never written back.
// HALF: fp16 block, 64-byte lines, 64-byte swizzle, LDS.64 (two-way conflicts as in the cp.async version).
// ============================================================================================
// CPW = 4: 8 warps x 4 columns (255 registers); CPW = 2: 16 warps x 2 columns (<= 128 registers, LDS.64)
template <int EPS, bool HALF, int CPW>
__global__ void __launch_bounds__(32 * (32 / CPW), 1)
    k_norm_syrk_cols_tma(const __grid_constant__ CUtensorMap tmA, int n, int E, int n2, int T256, int c0, float *K)
{
    static_assert(CPW == 4 || (CPW == 2 && !HALF), "2 columns per warp only for the fp32 block");
    constexpr int R = 4, EP = 32, MT = 2, NT = 4, NTHR = 32 * (32 / CPW);
    constexpr uint32_t BRICK = HALF ? 32768u : 65536u;
    constexpr uint32_t RING_BYTES = 196608u;   // 3 fp32 bricks; the fold buffer [32 columns][EP*EP] fp32 (128 KB) overlays it
    extern __shared__ __align__(1024) uint8_t cs_raw[];
    uint8_t *cs = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(cs_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t brick0 = smem_u32(cs);
    float *s_fold = reinterpret_cast<float *>(cs);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(cs + RING_BYTES);   // [3]
    uint64_t *empty_bar = full_bar + COLS_BRICKS;                          // [3]
    const int tid = threadIdx.x, warp = uniform_warp_idx(), lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int S_eps = (E / EPS) * EPS;
    const int e4 = E >> 2;
    const int nstrips = (n2 - c0 + 31) / 32;
    const int nsteps = (n + 15) / 16;

    if (tid == 0) {
        tma_prefetch_desc(&tmA);
        for (int b = 0; b < COLS_BRICKS; b++) {
            mbar_init(&full_bar[b], 1);
            mbar_init(&empty_bar[b], NTHR / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();

    // this lane's reads: line L0 = t + 4g (+ 32 sl + 128 r), 16-byte piece `warp` (fp32) / 8 bytes of piece warp/2 (fp16)
    const uint32_t L0 = (uint32_t)(t + 4 * g);
    const uint32_t rd_base = HALF ? L0 * 64u + ((((uint32_t)warp >> 1) ^ ((L0 >> 1) & 3u)) << 4) + ((uint32_t)warp & 1u) * 8u
                             : CPW == 4 ? L0 * 128u + ((((uint32_t)warp) ^ (L0 & 7u)) << 4)
                                        : L0 * 128u + ((((uint32_t)warp >> 1) ^ (L0 & 7u)) << 4) + ((uint32_t)warp & 1u) * 8u;
    constexpr uint32_t SL_STEP = HALF ? 2048u : 4096u, R_STEP = HALF ? 8192u : 16384u;

    uint32_t it = 0;          // running brick count of this CTA: slot = it % 3, use = it / 3
    uint32_t slot = 0, par = 0;   // slot / parity of brick `it`
    for (int strip = blockIdx.x; strip < nstrips; strip += gridDim.x) {
        const int j0 = c0 + strip * 32;
        const int tjx = (int)(j0 >> 8), jo = (int)(j0 & 255);
        // producer (one elected lane of warp 0): brick of row step st -> ring position idx
        auto issue = [&](int st, uint32_t idx) {
            const uint32_t sl = idx % COLS_BRICKS, use = idx / COLS_BRICKS;
            mbar_wait(&empty_bar[sl], (use & 1u) ^ 1u);       // every warp has released the slot's previous brick
            mbar_expect_tx(&full_bar[sl], BRICK);
            const int i0 = st * 16;
            tma_load_5d(&tmA, &full_bar[sl], brick0 + sl * BRICK, jo, 0, ((i0 >> 8) * T256 + tjx) * e4, (i0 & 255) >> 2, 0);
        };
        for (int seg0 = 0; seg0 < nsteps; seg0 += COLS_SEG_STEPS) {
            const int seg1 = seg0 + COLS_SEG_STEPS < nsteps ? seg0 + COLS_SEG_STEPS : nsteps;
            float acc[CPW][MT][NT][4];
#pragma unroll
            for (int c = 0; c < CPW; c++)
#pragma unroll
                for (int a = 0; a < MT; a++)
#pragma unroll
                    for (int b = 0; b < NT; b++)
#pragma unroll
                        for (int d = 0; d < 4; d++) acc[c][a][b][d] = 0.f;
            if (warp == 0) {
                if (elect_one_sync()) {
                    issue(seg0, it);
                    if (seg0 + 1 < seg1) issue(seg0 + 1, it + 1);
                }
                __syncwarp();
            }
            for (int st = seg0; st < seg1; st++) {
                if (warp == 0) {
                    if (st + 2 < seg1 && elect_one_sync()) issue(st + 2, it + 2);
                    __syncwarp();
                }
                mbar_wait(&full_bar[slot], par);
                // ---- this lane's 4 epochs x 4 rows x 4 columns
                float vals[R][4][CPW];
                const uint32_t bb = brick0 + slot * BRICK + rd_base;
#pragma unroll
                for (int r = 0; r < R; r++)
#pragma unroll
                    for (int sl = 0; sl < 4; sl++) {
                        if constexpr (HALF) {
                            const uint2 q = lds64(bb + (uint32_t)sl * SL_STEP + (uint32_t)r * R_STEP);
                            const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&q.x));
                            const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&q.y));
                            vals[r][sl][0] = lo.x, vals[r][sl][1] = lo.y, vals[r][sl][2] = hi.x, vals[r][sl][3] = hi.y;
                        } else if constexpr (CPW == 4) {
                            const uint4 q = lds128(bb + (uint32_t)sl * SL_STEP + (uint32_t)r * R_STEP);
                            vals[r][sl][0] = __uint_as_float(q.x), vals[r][sl][1] = __uint_as_float(q.y);
                            vals[r][sl][2] = __uint_as_float(q.z), vals[r][sl][3] = __uint_as_float(q.w);
                        } else {
                            const uint2 q = lds64(bb + (uint32_t)sl * SL_STEP + (uint32_t)r * R_STEP);
                            vals[r][sl][0] = __uint_as_float(q.x), vals[r][sl][1] = __uint_as_float(q.y);
                        }
                    }
                // the brick is in registers: hand the slot back to the producer
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[slot]);
                if (st * 16 + 16 > n) {   // ragged last row step (block-uniform): rows >= n hold stale scratch
#pragma unroll
                    for (int sl = 0; sl < 4; sl++)
                        if (st * 16 + 4 * sl + t >= n) {
#pragma unroll
                            for (int r = 0; r < R; r++)
#pragma unroll
                                for (int c = 0; c < CPW; c++) vals[r][sl][c] = 0.f;
                        }
                }
                // ---- within-subject z-score per (row, column), then K_j += Z Z^T per column
                zscore_frag<EPS, R, 4, CPW>([&](int r, int sl, int u) -> float & { return vals[r][sl][u]; }, g, S_eps);
#pragma unroll
                for (int c = 0; c < CPW; c++) mma_zzt(acc[c], [&](int r, int sl) { return vals[r][sl][c]; });
                it++;
                if (++slot == COLS_BRICKS) slot = 0, par ^= 1u;
            }
            // ---- fold the accumulators into K: registers -> smem [32 columns][EP*EP] -> mirrored, coalesced += on K.
            // Every brick of the segment has been consumed (no bulk copy is in flight), all warps are past their reads.
            __syncthreads();
#pragma unroll
            for (int c = 0; c < CPW; c++) store_frag(s_fold + (size_t)(warp * CPW + c) * (EP * EP), acc[c], g, t);
            __syncthreads();
            const int ncols = n2 - j0 < 32 ? n2 - j0 : 32;       // real columns of this strip
            // E % 4 == 0 here, and K + j0*E*E is 16-byte aligned whenever K is: always 16-byte read-modify-writes
            fold_strip<EP, NTHR, true, false>(K + (size_t)j0 * (E * E), s_fold, E, ncols);
            fence_proxy_async_smem();   // the fold's generic-proxy smem accesses are ordered before the next bulk copies
            __syncthreads();
        }
    }
}

__global__ void k_scale(float *x, long n, float s)
{
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        x[i] = s == 0.f ? 0.f : x[i] * s;
}

// eps_mode: 0 = plain SYRK of normalised data; > 0 = fused normalisation with that eps
static bool fused_supported(int E, int eps_mode)
{
    if (E > 64) return false;
    if (eps_mode == 0) return true;
    if (eps_mode & (eps_mode - 1)) return false;  // power of two only
    return eps_mode <= (E <= 32 ? 32 : 64);
}

// (stride_i, ld, chunk_step) describe where element (i, e, j) of the correlation block lives:
//   C[i*stride_i + e*ld + (j/256)*chunk_step + j%256]
// classic [nb][E][ld] layout: stride_i = E*ld, chunk_step = 256.  Tiled [nb/256][T256][E][256 i][256 j] layout
// (every 256x256 pair tile of the GEMM is one contiguous 256 KB run; the E tiles of one (row block, column
// block) are adjacent): stride_i = 256, ld = 65536, chunk_step = E*65536, and i -> (i/256)*T256*chunk_step +
// (i%256)*stride_i inside the kernel.
// rb_stride: elements between 256-row blocks of a tiled block when the kernel is given only a column RANGE of it (0: the
// range is the whole block); K64: optional fp64 accumulator [E][E] for sum_over_rows (then K is not touched)
static int launch_norm_syrk(const float *C, long nb, int E, long n2, long stride_i, long ld, int eps_mode,
                            int fisher_done, long self_col0, float beta, float *K, int sum_over_rows, cudaStream_t st,
                            long chunk_step = 256, int half_in = 0, long rb_stride = 0, double *K64 = nullptr)
{
    if (!fused_supported(E, eps_mode)) return fail(FCMA_EINVAL, "internal: fused norm+syrk unsupported E=%d eps=%d", E, eps_mode);
    if (sum_over_rows && !K64) {
        // K = beta*K, then atomically accumulate the per-row kernels
        k_scale<<<1, 256, 0, st>>>(K, (long)E * E, beta);
        LAUNCH_CHECK("k_scale");
    }
    const bool vec = ((ld & 3) == 0) && ((stride_i & 3) == 0) && (((uintptr_t)C & 15) == 0);
    if (!vec && chunk_step != 256) return fail(FCMA_EINVAL, "internal: tiled layout needs the vector path");
    const bool fisher = eps_mode > 0 && !fisher_done;
    if (half_in && (fisher || chunk_step == 256 || !vec))
        return fail(FCMA_EINVAL, "internal: the fp16 block is tiled and already Fisher-transformed");
    // rows cost the same: a static stride over 16 blocks per SM balances well
    long g = nb < 16L * g_sm_count ? nb : 16L * g_sm_count;
    int rc = FCMA_OK;
    // k_norm_syrk<R, EPS, FISHER, VEC> holds 8R padded epochs: it is built for EPS = 0 (plain SYRK) and every power of two
    // up to 8R
    auto run = [&](auto R, auto FISHER, auto VEC) {
        constexpr size_t smem = (VEC ? (size_t)8 * 2 * (VEC == 2 ? R : 2 * R) * 32 * sizeof(float4) : 0) +
                                (R <= 4 ? (size_t)8 * (8 * R) * (8 * R) * sizeof(float) : 0);
        auto go = [&](auto EPS) {
            rc = launch_kernel(k_norm_syrk<R, EPS, FISHER, VEC>, (unsigned)g, 256, smem, st, "k_norm_syrk", C, nb, E, n2,
                               stride_i, ld, chunk_step, self_col0, beta, K, sum_over_rows, rb_stride, K64);
        };
        if constexpr (R == 2) return with_int<0, 1, 2, 4, 8, 16>(eps_mode, go);
        else if constexpr (R == 4) return with_int<0, 1, 2, 4, 8, 16, 32>(eps_mode, go);
        else return with_int<0, 1, 2, 4, 8, 16, 32, 64>(eps_mode, go);
    };
    auto per_layout = [&](auto R) {   // VEC: 0 scalar loads, 1 cp.async of an fp32 block, 2 of an fp16 block
        if (half_in) return run(R, std::false_type{}, IntC<2>{});
        if (fisher) return vec ? run(R, std::true_type{}, IntC<1>{}) : run(R, std::true_type{}, IntC<0>{});
        return vec ? run(R, std::false_type{}, IntC<1>{}) : run(R, std::false_type{}, IntC<0>{});
    };
    bool ok;
    if (E <= 16 && eps_mode <= 16 && !half_in && !fisher && vec)
        // 16 padded epochs instead of 32 (lane = 2 epochs): half the statistics and MMA work per byte of the pipelines'
        // fp32 block (BASELINE configs[1]: E = 16)
        ok = run(IntC<2>{}, std::false_type{}, IntC<1>{});
    else
        ok = E <= 32 ? per_layout(IntC<4>{}) : per_layout(IntC<8>{});
    if (!ok) return fail(FCMA_EINVAL, "internal: no k_norm_syrk instantiation for E=%d eps=%d", E, eps_mode);
    return rc;
}

// column-direction pass over a tiled fp32 block (k_norm_syrk_cols): K[j] += ... for block columns [c0, n2)
static bool cols_supported(int E, int eps)
{
    return E <= 64 && eps >= 1 && eps <= (E <= 32 ? 32 : 64) && (eps & (eps - 1)) == 0;
}
static int launch_norm_syrk_cols(const void *A, long n, int E, long n2, long T256, long c0, int eps, float *K,
                                 cudaStream_t st, int half_in = 0, bool use_tma = false, bool v2 = false, bool pad32 = false)
{
    if (!cols_supported(E, eps) || (c0 & 31) || c0 >= n2) return fail(FCMA_EINVAL, "internal: column pass unsupported E=%d eps=%d c0=%ld", E, eps, c0);
    const float *A32 = reinterpret_cast<const float *>(A);
    int rc = FCMA_OK;
    if (E > 32) {   // 32 < E <= 64, fp32 block: one column per warp, 8-column strips (k_norm_syrk_cols64)
        if (half_in) return fail(FCMA_EINVAL, "internal: no column pass over an fp16 block for E=%d", E);
        const long nstrips8 = cdiv(n2 - c0, 8);
        const unsigned grid64 = (unsigned)(nstrips8 < g_sm_count ? nstrips8 : g_sm_count);
        const size_t smem64 = (size_t)8 * 64 * 64 * sizeof(float) + 128;   // the fold area; the 3 bricks (102 KB) lie inside it
        if (!with_int<1, 2, 4, 8, 16, 32, 64>(eps, [&](auto EPS) {
                rc = launch_kernel(k_norm_syrk_cols64<EPS>, grid64, 256, smem64, st, "k_norm_syrk_cols64", A32, n, E, n2, T256, c0, K);
            }))
            return fail(FCMA_EINVAL, "internal: no k_norm_syrk_cols64 instantiation for eps=%d", eps);
        return rc;
    }
    const long nstrips = cdiv(n2 - c0, 32);
    const unsigned grid = (unsigned)(nstrips < g_sm_count ? nstrips : g_sm_count);
    // FCMA_FLAG_COLS_TMA: TMA-fed bricks + mbarrier ring (k_norm_syrk_cols_tma) when the block can be described to TMA (E a
    // multiple of 4) and K allows 16-byte read-modify-writes.  It removes the 4096 LDGSTS per brick and the per-brick
    // bar.sync; opt-in, the cp.async kernel below stays the default.
    if (use_tma && (E & 3) == 0 && ((uintptr_t)K & 15) == 0 && ((uintptr_t)A & 15) == 0) {
        CUtensorMap tmA;
        rc = make_cols_map(&tmA, A, (size_t)cdiv(n, 256) * (size_t)T256, E, half_in);
        if (rc) return rc;
        const size_t smem_t = 196608 + 64 + 1024;
        auto go = [&](auto kernel) {
            rc = launch_kernel(kernel, grid, 256, smem_t, st, "k_norm_syrk_cols_tma", tmA, (int)n, E, (int)n2, (int)T256, (int)c0, K);
        };
        if (!with_int<1, 2, 4, 8, 16, 32>(eps, [&](auto EPS) {
                half_in ? go(k_norm_syrk_cols_tma<EPS, true, 4>) : go(k_norm_syrk_cols_tma<EPS, false, 4>);
            }))
            return fail(FCMA_EINVAL, "internal: no k_norm_syrk_cols_tma instantiation for eps=%d", eps);
        return rc;
    }
    // E <= 16 (fp32 block): 16-epoch bricks, two CTAs per SM (k_norm_syrk_cols16); the kernels below pad to 32 epochs
    if (!half_in && E <= 16 && eps <= 16 && !use_tma && !v2 && !pad32) {
        const size_t smem16 = (size_t)COLS_BRICKS * 32768 + 16384 + 128;
        const unsigned grid16 = (unsigned)(nstrips < 2L * g_sm_count ? nstrips : 2L * g_sm_count);
        if (!with_int<1, 2, 4, 8, 16>(eps, [&](auto EPS) {
                rc = launch_kernel(k_norm_syrk_cols16<EPS>, grid16, 256, smem16, st, "k_norm_syrk_cols16", A32, n, E, n2, T256, c0, K);
            }))
            return fail(FCMA_EINVAL, "internal: no k_norm_syrk_cols16 instantiation for eps=%d", eps);
        return rc;
    }
    // FCMA_FLAG_COLS_V2: thread-per-row normalisation, fp16 staging, ldmatrix fragments (k_norm_syrk_cols2, fp32 block).
    // ~2x fewer instructions than the fragment-layout kernel below; the column pass is bound by what it moves, not by
    // what it issues.  Opt-in, tested.
    if (!half_in && v2) {
        const size_t smem2 = (size_t)COLS_BRICKS * 65536 + 32768 + 1024;
        auto go = [&](auto kernel, unsigned threads) {
            rc = launch_kernel(kernel, grid, threads, smem2, st, "k_norm_syrk_cols2", A32, n, E, n2, T256, c0, K);
        };
        if (!with_int<1, 2, 4, 8, 16, 32>(eps, [&](auto EPS) {
#ifdef FCMA_DIAG
                // FCMA_COLS_V2_CPW=2: 16 warps x 2 columns (A/B)
                const char *cpw = diag_env("FCMA_COLS_V2_CPW");
                if (cpw && cpw[0] == '2') return go(k_norm_syrk_cols2<EPS, 2>, 512);
#endif
                go(k_norm_syrk_cols2<EPS, 4>, 256);
            }))
            return fail(FCMA_EINVAL, "internal: no k_norm_syrk_cols2 instantiation for eps=%d", eps);
        return rc;
    }
    // bricks (3 x 64 KB fp32 / 3 x 32 KB fp16); the fold buffer [32 columns][32*32] fp32 = 128 KB overlays them
    const size_t smem = (half_in ? (size_t)131072 : (size_t)COLS_BRICKS * 65536) + 1024;
    auto go = [&](auto kernel, unsigned threads) {
        rc = launch_kernel(kernel, grid, threads, smem, st, "k_norm_syrk_cols", A, n, E, n2, T256, c0, K);
    };
    if (!with_int<1, 2, 4, 8, 16, 32>(eps, [&](auto EPS) {
            if (half_in) return go(k_norm_syrk_cols<EPS, 4, true>, 256);
#ifdef FCMA_DIAG
            // 4 columns per warp (8 warps, 255 registers) by default; FCMA_COLS_CPW=2 selects 2 columns per warp (16 warps
            // at 128 registers, with spills and two-way conflicts on the 8-byte LDS; A/B)
            const char *cpw = diag_env("FCMA_COLS_CPW");
            if (cpw && cpw[0] == '2') return go(k_norm_syrk_cols<EPS, 2, false>, 512);
#endif
            go(k_norm_syrk_cols<EPS, 4, false>, 256);
        }))
        return fail(FCMA_EINVAL, "internal: no k_norm_syrk_cols instantiation for eps=%d", eps);
    return rc;
}

// ============================================================================================
// C ABI
// ============================================================================================
extern "C" int fcma_pack_operand(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e, int normalize,
                                 int precision, void *packed_dev, size_t packed_bytes, void *stream)
{
    return fcma_pack_operand_range(epochs_dev, E, T, V, ld, T_e, normalize, precision, 0, V, packed_dev, packed_bytes, stream);
}

static int pack_operand_impl(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e, int normalize,
                             int precision, long v_begin, long v_end, int e_begin, int e_count, void *packed_dev,
                             size_t packed_bytes, void *stream);
extern "C" int fcma_pack_operand_range(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e, int normalize,
                                       int precision, long v_begin, long v_end, void *packed_dev, size_t packed_bytes,
                                       void *stream)
{
    return pack_operand_impl(epochs_dev, E, T, V, ld, T_e, normalize, precision, v_begin, v_end, 0, E, packed_dev, packed_bytes, stream);
}
// voxels [v_begin, v_end) of epochs [e_begin, e_begin + e_count)
static int pack_operand_impl(const float *epochs_dev, int E, int T, long V, long ld, const int *T_e, int normalize,
                             int precision, long v_begin, long v_end, int e_begin, int e_count, void *packed_dev,
                             size_t packed_bytes, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    PrecInfo pi;
    if (!prec_info(precision, &pi)) return fail(FCMA_EINVAL, "unknown precision %d", precision);
    if (!epochs_dev || !packed_dev || E <= 0 || T <= 0 || V <= 0 || ld < V)
        return fail(FCMA_EINVAL, "fcma_pack_operand: bad arguments E=%d T=%d V=%ld ld=%ld", E, T, V, ld);
    if (v_begin < 0 || v_end > V || v_begin >= v_end)
        return fail(FCMA_EINVAL, "fcma_pack_operand_range: voxels [%ld, %ld) outside [0, %ld)", v_begin, v_end, V);
    if (e_begin < 0 || e_count <= 0 || e_begin + e_count > E) return fail(FCMA_EINVAL, "internal: bad epoch range for packing");
    size_t need = fcma_operand_bytes(precision, E, T, V);
    if (packed_bytes < need) return fail(FCMA_ENOMEM, "packed operand buffer too small: %zu < %zu", packed_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    AsyncBuf te_buf;
    int *d_Te = nullptr;
    if (T_e) {
        for (int e = 0; e < E; e++)
            if (T_e[e] <= 0 || T_e[e] > T) return fail(FCMA_EINVAL, "epoch %d has length %d outside (0, %d]", e, T_e[e], T);
        CUDA_TRY(te_buf.alloc(sizeof(int) * E, st));
        d_Te = static_cast<int *>(te_buf.p);
        CUDA_TRY(cudaMemcpyAsync(d_Te, T_e, sizeof(int) * E, cudaMemcpyHostToDevice, st));
    }
    const int Kp = fcma_operand_kp(precision, T);
    float *sd = reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(packed_dev) + operand_plane_bytes(pi, precision, E, T, V));
    dim3 grid((unsigned)cdiv(v_end - v_begin, 32), (unsigned)e_count);
    if (pi.pack == 0 && pi.planes == 1) k_pack_operand<0, 1><<<grid, 256, 0, st>>>(epochs_dev, E, T, V, ld, d_Te, normalize, packed_dev, Kp, sd, pi.in_scale, v_begin, v_end, e_begin);
    if (pi.pack == 0 && pi.planes == 2) k_pack_operand<0, 2><<<grid, 256, 0, st>>>(epochs_dev, E, T, V, ld, d_Te, normalize, packed_dev, Kp, sd, pi.in_scale, v_begin, v_end, e_begin);
    if (pi.pack == 1 && pi.planes == 1) k_pack_operand<1, 1><<<grid, 256, 0, st>>>(epochs_dev, E, T, V, ld, d_Te, normalize, packed_dev, Kp, sd, pi.in_scale, v_begin, v_end, e_begin);
    if (pi.pack == 1 && pi.planes == 2) k_pack_operand<1, 2><<<grid, 256, 0, st>>>(epochs_dev, E, T, V, ld, d_Te, normalize, packed_dev, Kp, sd, pi.in_scale, v_begin, v_end, e_begin);
    if (pi.pack == 2 && pi.planes == 2) k_pack_operand<2, 2><<<grid, 256, 0, st>>>(epochs_dev, E, T, V, ld, d_Te, normalize, packed_dev, Kp, sd, pi.in_scale, v_begin, v_end, e_begin);
    LAUNCH_CHECK("k_pack_operand");
    return FCMA_OK;   // te_buf is released in stream order by its destructor
}

extern "C" int fcma_epoch_normalize(float *epochs_dev, int E, int T, long V, long ld, const int *T_e, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!epochs_dev || E <= 0 || T <= 0 || V <= 0 || ld < V) return fail(FCMA_EINVAL, "fcma_epoch_normalize: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    AsyncBuf te_buf;
    int *d_Te = nullptr;
    if (T_e) {
        // a longer epoch would read (and overwrite) the next epoch's rows, or past the end for the last one
        for (int e = 0; e < E; e++)
            if (T_e[e] <= 0 || T_e[e] > T) return fail(FCMA_EINVAL, "epoch %d has length %d outside (0, %d]", e, T_e[e], T);
        CUDA_TRY(te_buf.alloc(sizeof(int) * E, st));
        d_Te = static_cast<int *>(te_buf.p);
        CUDA_TRY(cudaMemcpyAsync(d_Te, T_e, sizeof(int) * E, cudaMemcpyHostToDevice, st));
    }
    dim3 grid((unsigned)cdiv(V, 32), (unsigned)E);
    k_epoch_normalize<<<grid, 256, 0, st>>>(epochs_dev, T, V, ld, d_Te);
    LAUNCH_CHECK("k_epoch_normalize");
    return FCMA_OK;
}

extern "C" int fcma_corr_block(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                               long start, long nb, float *out_dev, long stride_i, long stride_e, int fisher_epochs,
                               void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!rows_op || !cols_op || !out_dev) return fail(FCMA_EINVAL, "fcma_corr_block: null pointer");
    return launch_corr_mma(rows_op, cols_op, precision, E, T, V, V2, start, nb, out_dev, stride_i, stride_e,
                            fisher_epochs, (cudaStream_t)stream);
}

extern "C" int fcma_corr_block_f32(const float *rows_epochs, long ldr, const float *cols_epochs, long ldc, int E, int T,
                                   long V, long V2, long start, long nb, float *out_dev, long stride_i, long stride_e,
                                   void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!rows_epochs || !cols_epochs || !out_dev || E <= 0 || T <= 0 || nb <= 0 || V2 <= 0 || start < 0 || start + nb > V)
        return fail(FCMA_EINVAL, "fcma_corr_block_f32: bad arguments");
    if (E > 65535 || cdiv(nb, 64) > 65535) return fail(FCMA_EINVAL, "fcma_corr_block_f32: block too large");
    dim3 grid((unsigned)cdiv(V2, 64), (unsigned)cdiv(nb, 64), (unsigned)E);
    k_corr_simt<<<grid, 256, 0, (cudaStream_t)stream>>>(rows_epochs, ldr, cols_epochs, ldc, T, V2, start, nb, out_dev,
                                                        stride_i, stride_e);
    LAUNCH_CHECK("k_corr_simt");
    return FCMA_OK;
}

extern "C" int fcma_within_subject_norm(float *corr_dev, long n0, int E, long n2, int eps, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!corr_dev || n0 <= 0 || E <= 0 || n2 <= 0) return fail(FCMA_EINVAL, "fcma_within_subject_norm: bad shape");
    if (eps <= 0) return fail(FCMA_EINVAL, "fcma_within_subject_norm: epochs_per_subj must be positive");
    if (E / eps == 0) return FCMA_OK;  // nSubjs == 0: nothing is touched (fcma_extension.cc:52-55)
    long total = n0 * (E / eps) * n2;
    long blocks = cdiv(total, 256);
    if (blocks > 148L * 64) blocks = 148L * 64;
    k_within_subject_norm<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(corr_dev, n0, E, n2, eps);
    LAUNCH_CHECK("k_within_subject_norm");
    return FCMA_OK;
}

static int launch_syrk_simt(const float *z, long nb, int E, long n2, long stride_i, long ld, float beta, float *K,
                            int sum_over_rows, cudaStream_t st)
{
    if (sum_over_rows) {
        k_scale<<<1, 256, 0, st>>>(K, (long)E * E, beta);
        LAUNCH_CHECK("k_scale");
    }
    size_t smem = (size_t)64 * (E + 1) * sizeof(float);
    if (smem > 200 * 1024) return fail(FCMA_EINVAL, "E=%d too large for the SIMT kernel-matrix path", E);
    long g = nb < 148L * 8 ? nb : 148L * 8;
    return launch_kernel(k_syrk_simt, (unsigned)g, 256, smem, st, "k_syrk_simt", z, nb, E, n2, stride_i, ld, beta, K,
                         sum_over_rows);
}

extern "C" int fcma_kernel_matrices(const float *z_dev, long nb, int E, long n2, long stride_i, long ld, float beta,
                                    float *K_dev, int sum_over_rows, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!z_dev || !K_dev || nb <= 0 || E <= 0 || n2 <= 0 || ld < n2) return fail(FCMA_EINVAL, "fcma_kernel_matrices: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (fused_supported(E, 0)) return launch_norm_syrk(z_dev, nb, E, n2, stride_i, ld, 0, 1, -1, beta, K_dev, sum_over_rows, st);
    return launch_syrk_simt(z_dev, nb, E, n2, stride_i, ld, beta, K_dev, sum_over_rows, st);
}

extern "C" int fcma_norm_kernel_matrices(const float *corr_dev, long nb, int E, long n2, long stride_i, long ld, int eps,
                                         int fisher_done, long self_col0, float beta, float *K_dev, int sum_over_rows,
                                         void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!corr_dev || !K_dev || nb <= 0 || E <= 0 || n2 <= 0 || ld < n2 || eps <= 0)
        return fail(FCMA_EINVAL, "fcma_norm_kernel_matrices: bad arguments");
    if (!fused_supported(E, eps))
        return fail(FCMA_EINVAL, "fused normalise+kernel needs E <= 64 and a power-of-two epochs_per_subj (E=%d eps=%d): "
                                 "use fcma_within_subject_norm + fcma_kernel_matrices", E, eps);
    return launch_norm_syrk(corr_dev, nb, E, n2, stride_i, ld, eps, fisher_done, self_col0, beta, K_dev, sum_over_rows,
                            (cudaStream_t)stream);
}

extern "C" size_t fcma_work_bytes_per_row(int E, long V2)
{
    // the fused pipelines store the block tiled as [rows/256][T256][E][256][256] (T256 = ceil(V2/256))
    return (size_t)E * round_up(V2, 256) * sizeof(float);
}

// Optional per-kernel timing of the fused pipelines (bench.py's live roofline measurement): when enabled,
// CUDA events bracket the GEMM and the normalise+SYRK launches on the launch stream.
static int g_timing_on = 0;
static double g_t_gemm = 0.0, g_t_syrk = 0.0, g_t_syrk2 = 0.0;   // syrk2: second normalise+SYRK launch of a symmetric pass
static long g_t_passes = 0;
extern "C" void fcma_timing_enable(int on)
{
    g_timing_on = on;
    g_t_gemm = g_t_syrk = g_t_syrk2 = 0.0;
    g_t_passes = 0;
}
extern "C" long fcma_timing_read3(double *gemm_ms, double *syrk_ms, double *syrk2_ms)
{
    if (gemm_ms) *gemm_ms = g_t_gemm;
    if (syrk_ms) *syrk_ms = g_t_syrk - g_t_syrk2;
    if (syrk2_ms) *syrk2_ms = g_t_syrk2;
    return g_t_passes;
}
extern "C" long fcma_timing_read(double *gemm_ms, double *syrk_ms)
{
    if (gemm_ms) *gemm_ms = g_t_gemm;
    if (syrk_ms) *syrk_ms = g_t_syrk;
    return g_t_passes;
}
// Events of one pipeline pass while timing is on (each call records one on `st`; all do nothing while it is off).  end()
// waits for the pass and adds GEMM = start..gemm_done, SYRK = gemm_done..end and, if rows_done() was called, SYRK2 =
// rows_done..end to the totals.
class PassTimer {
    EventSet<4> evs;   // start, GEMM done, end, rows done
    cudaStream_t st;
    bool rows = false;
    int record(int k)
    {
        if (evs.on) CUDA_TRY(cudaEventRecord(evs.ev[k], st));
        return FCMA_OK;
    }

public:
    explicit PassTimer(cudaStream_t s) : st(s) {}
    int start()
    {
        if (!g_timing_on) return FCMA_OK;
        CUDA_TRY(evs.create());
        return record(0);
    }
    int gemm_done() { return record(1); }
    int rows_done()
    {
        rows = true;
        return record(3);
    }
    int end()
    {
        if (!evs.on) return FCMA_OK;
        CUDA_TRY(cudaEventRecord(evs.ev[2], st));
        CUDA_TRY(cudaEventSynchronize(evs.ev[2]));
        float gemm = 0.f, syrk = 0.f, syrk2 = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&gemm, evs.ev[0], evs.ev[1]));
        CUDA_TRY(cudaEventElapsedTime(&syrk, evs.ev[1], evs.ev[2]));
        if (rows) CUDA_TRY(cudaEventElapsedTime(&syrk2, evs.ev[3], evs.ev[2]));
        g_t_gemm += gemm, g_t_syrk += syrk, g_t_syrk2 += syrk2, g_t_passes++;
        return FCMA_OK;
    }
};

// Fisher-z block of the fused pipelines in fp16 rather than fp32: FCMA_FLAG_F16_INTERMEDIATE asks for it, and the
// single-product reduced-precision operand modes (bf16 / tf32) take it by default.  The fp16 values' rounding errors are
// independent across the V2 columns the kernel matrix sums over: measured max|dK|/max|K| = 1.5e-5 at V2 = 50 000 (the
// reference's own fp32 ssyrk rounding noise is 1e-5), while both kernels move half the bytes (-8..12 % per step).  The
// fp32-faithful modes keep an fp32 block unless the flag asks otherwise; correlation values returned by fcma_corr_block
// are never rounded.  Diagnostic build: FCMA_F16_INTERMEDIATE=0|1 overrides (A/B).
static bool half_block(int precision, int flags)
{
    bool half = (flags & FCMA_FLAG_F16_INTERMEDIATE) || precision == FCMA_PREC_BF16 || precision == FCMA_PREC_TF32;
    const char *f16i = diag_env("FCMA_F16_INTERMEDIATE");
    if (f16i && (f16i[0] == '0' || f16i[0] == '1')) half = f16i[0] == '1';
    return half;
}

// Second stage of fcma_voxel_feature_kernels: the per-voxel fp64 kernel matrices of the normalised correlation vectors
// (k_norm_gram_f64) instead of the fp32 SYRK.  kind 0 linear, 1 rbf; outputs [nb][E][E].
struct FeatureStage {
    int kind;
    double gamma;
    double *K_fit, *K_pred;
};
static int launch_norm_gram_f64(const float *C, long nb, int E, long n2, long stride_i, long ld, long chunk_step, long t256,
                                int eps, int kind, double gamma, double *K_fit, double *K_pred, cudaStream_t st);

// shared body of the fused pipelines; with `feat` the GEMM writes raw r and the feature stage replaces normalise+SYRK
static int run_pipeline(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2, long start,
                        long nb, int eps, int flags, float *work, size_t work_bytes, float *K, int sum_over_rows,
                        cudaStream_t st, const FeatureStage *feat = nullptr)
{
    if (!rows_op || !cols_op || !work || !(K || feat)) return fail(FCMA_EINVAL, "pipeline: null pointer");
    if (nb <= 0 || start < 0 || start + nb > V) return fail(FCMA_EINVAL, "pipeline: rows [%ld, %ld) outside [0, %ld)", start, start + nb, V);
    if (eps < 0) return fail(FCMA_EINVAL, "pipeline: negative epochs_per_subj");
    if (((uintptr_t)work & 15)) return fail(FCMA_EINVAL, "pipeline: work buffer must be 16-byte aligned");
    const long ld = round_up(V2, 32);
    const size_t row_bytes = fcma_work_bytes_per_row(E, V2);   // >= E * ld * 4 (also covers the tiled layout)
    long rows_per_pass = (long)(work_bytes / row_bytes);
    if (rows_per_pass < 1) return fail(FCMA_ENOMEM, "work buffer too small: %zu bytes < %zu per row", work_bytes, row_bytes);
    if (rows_per_pass > 256) rows_per_pass = (rows_per_pass / 256) * 256;  // whole GEMM tiles
    // Classifier semantics: eps <= 1 -> no normalisation at all (classifier.py:204)
    const bool normalise = sum_over_rows ? eps > 1 : eps >= 1;
    const bool fused = normalise ? fused_supported(E, eps) : fused_supported(E, 0);
    const int S_eps = normalise ? (E / eps) * eps : 0;
    const bool fisher_in_gemm = !feat && normalise && fused && !(flags & FCMA_FLAG_FISHER_IN_PASS2);
    const bool mask_self = (flags & FCMA_FLAG_MASK_SELF) != 0;
    if (mask_self && (feat || !(normalise && fused)))
        return fail(FCMA_EINVAL, "FCMA_FLAG_MASK_SELF needs the fused normalise+kernel path (E <= 64, power-of-two eps)");
    // Tiled intermediate [n/256][T256][E][256][256]: every 256x256 pair tile of the GEMM is one contiguous 256 KB
    // run and the E tiles of one (row block, column block) are adjacent, so the fused normalise+SYRK kernel reads
    // row i as E runs of 1 KB, 256 KB apart, inside one 8 MB region.  Needs whole 256-row blocks of workspace.
    // FCMA_FLAG_STRIDED_BLOCK keeps the strided [i][e][j] block.
    const long t256 = cdiv(V2, 256);
    const bool tiled = !(flags & FCMA_FLAG_STRIDED_BLOCK) && (fused || feat) && V2 < (1L << 31) && rows_per_pass >= 256;
    // an fp16 block needs the tiled layout and holds Fisher-z values (applied in the GEMM epilogue)
    const bool half16 = half_block(precision, flags) && tiled && normalise && fisher_in_gemm;
    for (long done = 0; done < nb; done += rows_per_pass) {
        const long n = nb - done < rows_per_pass ? nb - done : rows_per_pass;
        PassTimer timer(st);
        int rc = timer.start();
        if (rc) return rc;
        if (tiled)
            rc = launch_corr_mma(rows_op, cols_op, precision, E, T, V, V2, start + done, n, work, 4, 4,
                                  fisher_in_gemm ? S_eps : 0, st, t256, half16 ? 1 : 0);
        else
            rc = launch_corr_mma(rows_op, cols_op, precision, E, T, V, V2, start + done, n, work, (long)E * ld, ld,
                                  fisher_in_gemm ? S_eps : 0, st);
        if (rc) return rc;
        rc = timer.gemm_done();
        if (rc) return rc;
        float *Kdst = sum_over_rows ? K : K + (size_t)done * E * E;
        const float beta = sum_over_rows ? 1.0f : 0.0f;
        if (feat) {
            const size_t off = (size_t)done * E * E;
            rc = tiled ? launch_norm_gram_f64(work, n, E, V2, 256, 65536, (long)E * 65536, t256, eps, feat->kind, feat->gamma,
                                              feat->K_fit + off, feat->K_pred ? feat->K_pred + off : nullptr, st)
                       : launch_norm_gram_f64(work, n, E, V2, (long)E * ld, ld, 256, t256, eps, feat->kind, feat->gamma,
                                              feat->K_fit + off, feat->K_pred ? feat->K_pred + off : nullptr, st);
        } else if (tiled) {
            rc = launch_norm_syrk(work, n, E, V2, 256, 65536, normalise ? eps : 0, (normalise && fisher_in_gemm) ? 1 : 0,
                                  mask_self ? start + done : -1, beta, Kdst, sum_over_rows, st, (long)E * 65536,
                                  half16 ? 1 : 0);
        } else if (normalise && fused) {
            rc = launch_norm_syrk(work, n, E, V2, (long)E * ld, ld, eps, fisher_in_gemm ? 1 : 0,
                                  mask_self ? start + done : -1, beta, Kdst, sum_over_rows, st);
        } else {
            if (normalise) {
                // generic-eps path: normalise the padded block [n][E][ld] in place (the pad columns hold
                // don't-care values that the kernel-matrix stage never reads: it is bounded by n2 = V2)
                long total = n * (E / eps) * ld;
                if (total > 0) {
                    long blocks = cdiv(total, 256);
                    if (blocks > 148L * 64) blocks = 148L * 64;
                    k_within_subject_norm<<<(unsigned)blocks, 256, 0, st>>>(work, n, E, ld, eps);
                    LAUNCH_CHECK("k_within_subject_norm");
                }
            }
            if (fused_supported(E, 0))
                rc = launch_norm_syrk(work, n, E, V2, (long)E * ld, ld, 0, 1, -1, beta, Kdst, sum_over_rows, st);
            else
                rc = launch_syrk_simt(work, n, E, V2, (long)E * ld, ld, beta, Kdst, sum_over_rows, st);
        }
        if (rc) return rc;
        rc = timer.end();
        if (rc) return rc;
    }
    return FCMA_OK;
}

// Symmetric pipeline for self-correlation (raw_data2 is None): corr[i][e][j] == corr[j][e][i], so only the
// blocks on and above the diagonal are contracted.  Pass p takes rows I = [a, a+n) against columns [a, V):
//   GEMM (symmetric mode)  -> A = tiled block rows I x columns [a, V)      (diagonal n x n part: upper tiles
//                                computed, lower tiles mirrored)
//                          -> B = tiled block rows [a+n, V) x columns I   (transposed copies)
//   normalise+SYRK over A  -> K[i] += sum_{j >= a} z z^T          for i in I
//   normalise+SYRK over B  -> K[j] += sum_{i in I} z z^T          for j in [a+n, V)
// After all passes of all callers (ranks) every K[x] has received every column exactly once.  Half the MMAs and
// half the Fisher transforms of the plain pipeline; HBM traffic per correlation is unchanged.
// which variant run_pipeline_sym takes for the column voxels' sums: 1 = column-direction pass over block A
// (E <= 32, power-of-two eps <= 32; fp32 or fp16 block), 0 = transposed block B + row pass
static bool sym_uses_cols(int precision, int E, int eps, int flags)
{
    if (flags & FCMA_FLAG_SYM_TRANSPOSED) return false;
    // 32 < E <= 64: the column kernel (fp32 block only) is opt-in; it halves the scratch per block row
    if (E > 32 && (half_block(precision, flags) || !(flags & FCMA_FLAG_COLS_WIDE))) return false;
    return cols_supported(E, eps);
}
// scratch per block row of a symmetric pass over rows [start, V): block A needs E * round_up(V - start, 256) floats per
// row; a transposed block B at most the same again
static size_t sym_row_bytes(int precision, int E, int eps, int flags, long V, long start)
{
    return (sym_uses_cols(precision, E, eps, flags) ? 1 : 2) * fcma_work_bytes_per_row(E, V - start);
}
extern "C" int fcma_sym_uses_column_pass(int precision, int E, int eps, int flags)
{
    return sym_uses_cols(precision, E, eps, flags) ? 1 : 0;
}

// Hooks of the host-buffer entry point (fcma_host_voxel_kernels_sym): the first pass' GEMM runs epoch group by epoch group
// as the groups arrive from the host (a GEMM tile needs only its own epoch), and the kernels of a pass are read back while the
// next pass computes (K rows [a, a+n) are final once the pass' row kernel has run).
struct SymHostHooks {
    int ngroups = 0;
    const int *e0 = nullptr, *cnt = nullptr;                  // epoch groups of the upload
    int (*prepare)(void *ctx, int g, cudaStream_t st) = nullptr;   // make group g's packed operand available on `st`
    void *ctx = nullptr;
    cudaStream_t copy = nullptr;                              // read-back stream
    float *K_host = nullptr;
    bool two_buffers = false;                                 // `work` may be split in two blocks: two passes follow the upload
};

static int run_pipeline_sym(const void *op, int precision, int E, int T, long V, long start, long nb, int eps, int flags,
                            float *work, size_t work_bytes, float *K, cudaStream_t st, const SymHostHooks *hooks = nullptr)
{
    if (!op || !work || !K) return fail(FCMA_EINVAL, "pipeline: null pointer");
    if (nb <= 0 || start < 0 || start + nb > V) return fail(FCMA_EINVAL, "pipeline: rows [%ld, %ld) outside [0, %ld)", start, start + nb, V);
    if (eps < 1) return fail(FCMA_EINVAL, "pipeline: epochs_per_subj must be positive");
    if (((uintptr_t)work & 15)) return fail(FCMA_EINVAL, "pipeline: work buffer must be 16-byte aligned");
    if (!fused_supported(E, eps)) return fail(FCMA_EINVAL, "symmetric pipeline needs the fused normalise+kernel path (E <= 64, power-of-two eps)");
    if ((nb & 255) && start + nb != V)
        return fail(FCMA_EINVAL, "symmetric pipeline: the row count must be a multiple of 256 unless the rows end at V");
    if (flags & FCMA_FLAG_FISHER_IN_PASS2) return fail(FCMA_EINVAL, "symmetric pipeline applies Fisher-z in the GEMM epilogue");
    const bool mask_self = (flags & FCMA_FLAG_MASK_SELF) != 0;
    const int S_eps = (E / eps) * eps;
    const bool half16 = half_block(precision, flags);
    const size_t esz = half16 ? sizeof(__half) : sizeof(float);
    // column-direction pass (E <= 32; fp32 or fp16 block): the column voxels' sums are taken from block A itself, no
    // transposed copy is stored.  FCMA_FLAG_SYM_TRANSPOSED keeps the transposed block B.
    const bool use_cols = sym_uses_cols(precision, E, eps, flags);
    const size_t row_bytes = sym_row_bytes(precision, E, eps, flags, V, start);
    // host-buffer mode with room for two blocks: the first TWO passes' GEMMs follow the upload group by group
    const bool grouped = hooks && hooks->ngroups > 0;
    const bool two = grouped && hooks->two_buffers && work_bytes / 2 / row_bytes >= 256;
    const size_t buf_bytes = two ? (work_bytes / 2) & ~(size_t)255 : work_bytes;
    long rows_per_pass = (long)(buf_bytes / row_bytes) & ~255L;
    if (rows_per_pass < 256)
        return fail(FCMA_ENOMEM, "work buffer too small for the symmetric pipeline: %zu bytes < %zu (256 rows)", work_bytes, 256 * row_bytes);
    const long npass = cdiv(nb, rows_per_pass);
    struct Pass {
        long a, n, colsA, t256, nt, rowsB;
    };
    auto geometry = [&](long p) {
        Pass g;
        g.a = start + p * rows_per_pass;
        g.n = nb - p * rows_per_pass < rows_per_pass ? nb - p * rows_per_pass : rows_per_pass;
        g.colsA = V - g.a, g.t256 = cdiv(g.colsA, 256), g.nt = cdiv(g.n, 256), g.rowsB = V - g.a - g.n;
        return g;
    };
    auto blockB = [&](const Pass &g, float *A) {
        return reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(A) + (size_t)g.nt * g.t256 * E * 65536 * esz);
    };
    auto gemm_pass = [&](const Pass &g, float *A, int e_begin, int e_count, bool fixup) -> int {
        if ((size_t)((g.nt * g.t256 + (use_cols ? 0 : (g.t256 - g.nt) * g.nt)) * E) * 65536 * esz > buf_bytes)
            return fail(FCMA_ENOMEM, "internal: symmetric pass does not fit the work buffer");
        SymOut so{use_cols ? nullptr : blockB(g, A)};
        return launch_corr_mma(op, op, precision, E, T, V, V, g.a, g.n, A, 4, 4, S_eps, st, g.t256, half16 ? 1 : 0, &so,
                                e_begin, e_count, fixup);
    };
    // normalise + SYRK of one pass: rows of the block, then its columns (or the rows of the transposed copy)
    auto syrk_pass = [&](const Pass &g, float *A, PassTimer *timer) -> int {
        int rc = launch_norm_syrk(A, g.n, E, g.colsA, 256, 65536, eps, 1, mask_self ? 0 : -1, 1.0f, K + (size_t)g.a * E * E, 0,
                                  st, (long)E * 65536, half16 ? 1 : 0);
        if (rc) return rc;
        if (timer && (rc = timer->rows_done())) return rc;
        if (hooks && hooks->K_host) {
            // rows [a, a+n) of K are final now (the columns left of this pass arrived through earlier column passes)
            EventSet<1> rowdone;
            CUDA_TRY(rowdone.create());
            CUDA_TRY(cudaEventRecord(rowdone.ev[0], st));
            CUDA_TRY(cudaStreamWaitEvent(hooks->copy, rowdone.ev[0], 0));
            CUDA_TRY(cudaMemcpyAsync(hooks->K_host + (size_t)g.a * E * E, K + (size_t)g.a * E * E,
                                     (size_t)g.n * E * E * sizeof(float), cudaMemcpyDeviceToHost, hooks->copy));
        }
        if (g.rowsB > 0 && use_cols)
            return launch_norm_syrk_cols(A, g.n, E, g.colsA, g.t256, g.n, eps, K + (size_t)g.a * E * E, st, half16 ? 1 : 0,
                                         (flags & FCMA_FLAG_COLS_TMA) != 0, (flags & FCMA_FLAG_COLS_V2) != 0,
                                         (flags & FCMA_FLAG_COLS_PAD32) != 0);
        if (g.rowsB > 0)
            return launch_norm_syrk(blockB(g, A), g.rowsB, E, g.n, 256, 65536, eps, 1, -1, 1.0f,
                                    K + (size_t)(g.a + g.n) * E * E, 0, st, (long)E * 65536, half16 ? 1 : 0);
        return FCMA_OK;
    };
    float *buf0 = work;
    float *buf1 = reinterpret_cast<float *>(reinterpret_cast<uint8_t *>(work) + buf_bytes);
    long first = 0;
    if (grouped) {
        // one GEMM launch per uploaded epoch group (a tile needs only its own epoch), the diagonal fix-up after the last
        const long ahead = (two && npass > 1) ? 2 : 1;
        for (int gi = 0; gi < hooks->ngroups; gi++) {
            int rc = hooks->prepare(hooks->ctx, gi, st);
            for (long p = 0; p < ahead && !rc; p++)
                rc = gemm_pass(geometry(p), p == 0 ? buf0 : buf1, hooks->e0[gi], hooks->cnt[gi], gi == hooks->ngroups - 1);
            if (rc) return rc;
        }
        for (long p = 0; p < ahead; p++) {
            int rc = syrk_pass(geometry(p), p == 0 ? buf0 : buf1, nullptr);
            if (rc) return rc;
        }
        first = ahead;
    }
    for (long p = first; p < npass; p++) {
        const Pass g = geometry(p);
        PassTimer timer(st);
        int rc = timer.start();
        if (rc) return rc;
        rc = gemm_pass(g, buf0, 0, E, true);
        if (rc) return rc;
        rc = timer.gemm_done();
        if (rc) return rc;
        rc = syrk_pass(g, buf0, &timer);
        if (rc) return rc;
        rc = timer.end();
        if (rc) return rc;
    }
    return FCMA_OK;
}

// Classifier kernel of ONE mask (a9 -> a10 -> a11, classifier.py:279-348) on the symmetric GEMM:  sum over ALL voxel pairs
//     K = sum_i sum_j z(i,:,j) z(i,:,j)^T,   z(i,:,j) == z(j,:,i)
// needs every pair once, so per pass  K += rowpass(diagonal square: holds (i,j) AND (j,i)) + 2 * rowpass(columns right of it)
// -- no column-direction pass and no transposed copy at all (a third less traffic than summing the per-voxel kernels).
// The two parts accumulate in fp64 (device atomics) and are combined at the end.
__global__ void k_classifier_combine(const double *S, int EE, float *K)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < EE) K[idx] += (float)(S[idx] + 2.0 * S[EE + idx]);
}
static int run_classifier_sym(const void *op, int precision, int E, int T, long V, int eps, int flags, float *work,
                              size_t work_bytes, float *K, cudaStream_t st)
{
    if (!op || !work || !K) return fail(FCMA_EINVAL, "pipeline: null pointer");
    if (eps < 2 || !fused_supported(E, eps)) return fail(FCMA_EINVAL, "symmetric classifier kernel needs the fused path (E <= 64, power-of-two eps >= 2)");
    const bool mask_self = (flags & FCMA_FLAG_MASK_SELF) != 0;
    const int S_eps = (E / eps) * eps;
    const bool half16 = half_block(precision, flags);
    const size_t esz = half16 ? sizeof(__half) : sizeof(float);
    const size_t row_bytes = fcma_work_bytes_per_row(E, V);
    const long rows_per_pass = (long)(work_bytes / row_bytes) & ~255L;
    if (rows_per_pass < 256) return fail(FCMA_ENOMEM, "work buffer too small for the symmetric pipeline");
    AsyncBuf sums;
    CUDA_TRY(sums.alloc(sizeof(double) * 2 * E * E, st));
    CUDA_TRY(cudaMemsetAsync(sums.p, 0, sizeof(double) * 2 * E * E, st));
    double *S = static_cast<double *>(sums.p);
    for (long a = 0; a < V; a += rows_per_pass) {
        const long n = V - a < rows_per_pass ? V - a : rows_per_pass;
        const long colsA = V - a, t256 = cdiv(colsA, 256), nt = cdiv(n, 256);
        if ((size_t)(nt * t256 * E) * 65536 * esz > work_bytes) return fail(FCMA_ENOMEM, "internal: symmetric pass does not fit the work buffer");
        SymOut so{nullptr};
        PassTimer timer(st);
        int rc = timer.start();
        if (rc) return rc;
        rc = launch_corr_mma(op, op, precision, E, T, V, V, a, n, work, 4, 4, S_eps, st, t256, half16 ? 1 : 0, &so);
        if (rc) return rc;
        rc = timer.gemm_done();
        if (rc) return rc;
        const long rb = t256 * (long)E * 65536;                       // elements between the 256-row blocks of the block
        const long sq = nt * 256 < colsA ? nt * 256 : colsA;          // columns of the diagonal square
        rc = launch_norm_syrk(work, n, E, sq, 256, 65536, eps, 1, mask_self ? 0 : -1, 1.0f, K, 1, st, (long)E * 65536,
                              half16 ? 1 : 0, rb, S);
        if (rc) return rc;
        if (colsA > sq) {
            const float *rest = half16 ? reinterpret_cast<const float *>(reinterpret_cast<const __half *>(work) + (size_t)nt * E * 65536)
                                       : work + (size_t)nt * E * 65536;
            rc = launch_norm_syrk(rest, n, E, colsA - sq, 256, 65536, eps, 1, -1, 1.0f, K, 1, st, (long)E * 65536,
                                  half16 ? 1 : 0, rb, S + (size_t)E * E);
            if (rc) return rc;
        }
        rc = timer.end();
        if (rc) return rc;
    }
    k_classifier_combine<<<(unsigned)cdiv((long)E * E, 256), 256, 0, st>>>(S, E * E, K);
    LAUNCH_CHECK("k_classifier_combine");
    return FCMA_OK;
}

extern "C" int fcma_classifier_kernel_sym(const void *op, int precision, int E, int T, long V, int eps, int flags,
                                          float *work_dev, size_t work_bytes, float *K_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    return run_classifier_sym(op, precision, E, T, V, eps, flags, work_dev, work_bytes, K_dev, (cudaStream_t)stream);
}

extern "C" long fcma_sym_rows_per_pass(int precision, int E, int eps, int flags, long V, long start, size_t work_bytes)
{
    const size_t row_bytes = sym_row_bytes(precision, E, eps, flags, V, start);
    return row_bytes ? (long)(work_bytes / row_bytes) & ~255L : 0;
}

extern "C" int fcma_voxel_kernels_sym(const void *op, int precision, int E, int T, long V, long start, long nb, int eps,
                                      int flags, float *work_dev, size_t work_bytes, float *K_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    return run_pipeline_sym(op, precision, E, T, V, start, nb, eps, flags, work_dev, work_bytes, K_dev, (cudaStream_t)stream);
}

// fcma_voxel_kernels_sym for epochs that are still ARRIVING (multi-GPU input exchange, exchange.py): the epochs come in
// `ngroups` contiguous groups, ready_events[g] (cudaEvent_t) fires when group g is complete in epochs_dev.  The library
// packs each group (voxels [start, V) only) as soon as its event has fired and runs the GEMMs of the first pass -- of the
// first two passes if `work` holds two blocks -- group by group, so that the upload hides under them; everything else
// follows as in fcma_voxel_kernels_sym.  Same results.
struct GroupedCtx {
    const float *epochs;
    int E, T;
    long V, start;
    const int *T_e;
    int normalize, precision;
    void *op;
    size_t opb;
    const int *e0, *cnt;
    void *const *ready;
};
static int grouped_prepare(void *vctx, int g, cudaStream_t st)
{
    GroupedCtx *c = static_cast<GroupedCtx *>(vctx);
    if (c->ready && c->ready[g]) CUDA_TRY(cudaStreamWaitEvent(st, (cudaEvent_t)c->ready[g], 0));
    return pack_operand_impl(c->epochs, c->E, c->T, c->V, c->V, c->T_e, c->normalize, c->precision, c->start, c->V, c->e0[g],
                             c->cnt[g], c->op, c->opb, st);
}
extern "C" int fcma_voxel_kernels_sym_grouped(const float *epochs_dev, const int *T_e, int normalize, void *op_dev,
                                              size_t op_bytes, int precision, int E, int T, long V, long start, long nb,
                                              int eps, int flags, int ngroups, const int *e0, const int *cnt,
                                              void *const *ready_events, float *work_dev, size_t work_bytes, float *K_dev,
                                              void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!epochs_dev || !op_dev || !e0 || !cnt || ngroups < 1 || ngroups > 64)
        return fail(FCMA_EINVAL, "fcma_voxel_kernels_sym_grouped: bad arguments");
    int next = 0;
    for (int g = 0; g < ngroups; g++) {
        if (e0[g] != next || cnt[g] <= 0) return fail(FCMA_EINVAL, "epoch groups must be contiguous and cover [0, E)");
        next += cnt[g];
    }
    if (next != E) return fail(FCMA_EINVAL, "epoch groups must be contiguous and cover [0, E)");
    if (op_bytes < fcma_operand_bytes(precision, E, T, V)) return fail(FCMA_ENOMEM, "packed operand buffer too small");
    GroupedCtx ctx{epochs_dev, E, T, V, start, T_e, normalize, precision, op_dev, op_bytes, e0, cnt, ready_events};
    SymHostHooks hooks;
    hooks.ngroups = ngroups, hooks.e0 = e0, hooks.cnt = cnt, hooks.prepare = grouped_prepare, hooks.ctx = &ctx;
    hooks.two_buffers = true;
    return run_pipeline_sym(op_dev, precision, E, T, V, start, nb, eps, flags, work_dev, work_bytes, K_dev, (cudaStream_t)stream,
                            &hooks);
}

extern "C" int fcma_voxel_kernels(const void *rows_op, const void *cols_op, int precision, int E, int T, long V, long V2,
                                  long start, long nb, int eps, int flags, float *work_dev, size_t work_bytes,
                                  float *K_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (eps <= 0) return fail(FCMA_EINVAL, "fcma_voxel_kernels: epochs_per_subj must be positive");
    return run_pipeline(rows_op, cols_op, precision, E, T, V, V2, start, nb, eps, flags, work_dev, work_bytes, K_dev, 0,
                        (cudaStream_t)stream);
}

extern "C" int fcma_classifier_kernel(const void *rows_op, const void *cols_op, int precision, int E, int T, long V,
                                      long V2, long start, long nb, int eps, int flags, float *work_dev,
                                      size_t work_bytes, float *K_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    return run_pipeline(rows_op, cols_op, precision, E, T, V, V2, start, nb, eps, flags, work_dev, work_bytes, K_dev, 1,
                        (cudaStream_t)stream);
}

extern "C" int fcma_gemm_nt(const float *A_dev, const float *B_dev, float *C_dev, long M, long N, long K, long lda,
                            long ldb, long ldc, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!A_dev || !B_dev || !C_dev || M <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || ldc < N)
        return fail(FCMA_EINVAL, "fcma_gemm_nt: bad arguments");
    if (cdiv(M, 64) > 65535) return fail(FCMA_EINVAL, "fcma_gemm_nt: M too large");
    dim3 grid((unsigned)cdiv(N, 64), (unsigned)cdiv(M, 64));
    k_gemm_nt<<<grid, 256, 0, (cudaStream_t)stream>>>(A_dev, B_dev, C_dev, M, N, K, lda, ldb, ldc);
    LAUNCH_CHECK("k_gemm_nt");
    return FCMA_OK;
}

extern "C" int fcma_row_normalize(float *X_dev, long R, long D, long ld, int nan_to_zero, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!X_dev || R <= 0 || D <= 0 || ld < D) return fail(FCMA_EINVAL, "fcma_row_normalize: bad arguments");
    long g = R < 148L * 8 ? R : 148L * 8;
    k_row_normalize<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(X_dev, R, D, ld, nan_to_zero);
    LAUNCH_CHECK("k_row_normalize");
    return FCMA_OK;
}


// ============================================================================================
// a7 tail + a8 on the GPU: decimal shrink and batched SVM cross-validation on precomputed kernels
// ============================================================================================
// Decimal shrink of voxelselector.py:409-412 / classifier.py:343-347, one warp per [E][E] kernel:
//   nd = len(str(int(K[0][0]))); if nd > 2: K *= 10**(2-nd)   (float32 multiply, like numpy)
// The digits of int(K00) are counted on the float itself, over its whole range (up to 39 digits): for an integer N,
// trunc(|f|) >= N <=> |f| >= N, and for N = 10^k that holds exactly when |f| >= the smallest float32 >= 10^k (the table,
// generated with Python integers and checked by tests/test_gpu_pack_and_side_kernels.py).  A negative value with
// int() != 0 adds one for the '-' sign.  NaN and +-inf, where the reference's int() raises, give nd = 1: K untouched.
__global__ void __launch_bounds__(128) k_shrink_kernels(float *K, long nv, int E, int *digits_out)
{
    constexpr float kPow10Ceil[38] = {
        0x1.400000p+3f, 0x1.900000p+6f, 0x1.f40000p+9f, 0x1.388000p+13f, 0x1.86a000p+16f, 0x1.e84800p+19f,
        0x1.312d00p+23f, 0x1.7d7840p+26f, 0x1.dcd650p+29f, 0x1.2a05f2p+33f, 0x1.748770p+36f, 0x1.d1a94cp+39f,
        0x1.2309d0p+43f, 0x1.6bcc42p+46f, 0x1.c6bf54p+49f, 0x1.1c3794p+53f, 0x1.63457ap+56f, 0x1.bc16d8p+59f,
        0x1.158e48p+63f, 0x1.5af1d8p+66f, 0x1.b1ae4ep+69f, 0x1.0f0cf2p+73f, 0x1.52d02ep+76f, 0x1.a78438p+79f,
        0x1.08b2a4p+83f, 0x1.4adf4cp+86f, 0x1.9d9720p+89f, 0x1.027e74p+93f, 0x1.431e10p+96f, 0x1.93e594p+99f,
        0x1.f8defap+102f, 0x1.3b8b5cp+106f, 0x1.8a6e34p+109f, 0x1.ed09c0p+112f, 0x1.342618p+116f, 0x1.812f9ep+119f,
        0x1.e17b86p+122f, 0x1.2ced34p+126f,
    };  // kPow10Ceil[k - 1] = smallest float32 >= 10^k
    const long v = (long)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (v >= nv) return;
    float *Kv = K + (size_t)v * E * E;
    const float k00 = Kv[0];
    int nd = 1;
    if (isfinite(k00)) {
        const float a = fabsf(k00);
#pragma unroll
        for (int k = 0; k < 38; k++) nd += a >= kPow10Ceil[k];
        if (k00 <= -1.0f) nd++;         // the '-' sign counts in len(str(.)); int(-0.5) is 0
    }
    if (digits_out && lane == 0) digits_out[v] = nd;
    if (nd > 2) {
        const float prop = (float)pow(10.0, (double)(2 - nd));   // float32(10**(2-nd))
        for (int idx = lane; idx < E * E; idx += 32) Kv[idx] *= prop;
    }
}

// Batched C-SVC cross-validation on precomputed kernels: one warp per (voxel, fold).
// The solver restates libsvm's SMO exactly as scikit-learn 1.9.0 runs it for
// SVC(kernel='precomputed') (sklearn/svm/src/libsvm/svm.cpp: Solver::Solve :665-925,
// select_working_set :946-1043 (WSS2, ">=" / "<=" tie-breaking = last index), calculate_rho
// :1126-1162, float Q values, double gradient, eps = tol, TAU = 1e-12; classes grouped with the
// smaller label first = +1 (svm_group_classes :2246-2326); prediction dec > 0 -> first class
// :2842-2905), with or without the shrinking heuristic (a template switch of k_svm_cv).  Lane l owns
// training samples l and l+32 (n_train <= 64).
struct SvmFold {
    int n_train, n_pos, n_test, pad;
    int train_idx[64];        // class (+1) samples first, original order inside a class
    int test_idx[64];
    unsigned char test_pos[64];
};

// A warp's staging area in the shrinking solver: do_shrinking moves the items' state between positions through it
struct SvmStage {
    double d[4][64];          // G, G_bar, alpha, QD by position
    int i[2][64];             // pm, y > 0
    unsigned char map[64];    // map[new position] = old position
};
// Dynamic shared memory of a k_svm_cv block (4 warps): the warps' Q [64][64] floats, then with shrinking their stages
constexpr int SVM_Q_FLOATS = 4 * 64 * 64;
constexpr size_t svm_smem_bytes(bool shrink)
{
    return SVM_Q_FLOATS * sizeof(float) + (shrink ? 4 * sizeof(SvmStage) : 0);
}

__device__ __forceinline__ void warp_argbest(double &val, int &idx, bool want_max)
{
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        double ov = __shfl_xor_sync(0xffffffffu, val, off);
        int oi = __shfl_xor_sync(0xffffffffu, idx, off);
        bool better = want_max ? (ov > val) : (ov < val);
        if (better || (ov == val && oi > idx)) {   // ties: the later index wins (">=" / "<=" scans)
            val = ov;
            idx = oi;
        }
    }
}

// The value at position pos of an array held lane-slot-wise (lane l holds positions l and l + 32), on every lane
template <typename T>
__device__ __forceinline__ T warp_at(const T (&a)[2], int pos)
{
    return __shfl_sync(0xffffffffu, (pos >> 5) ? a[1] : a[0], pos & 31);
}

// libsvm's analytic two-variable step with its clipping order (Solver::Solve, "update alpha[i] and alpha[j]")
__device__ __forceinline__ void smo_pair_update(double &ai, double &aj, double yi, double yj, double QDi, double QDj,
                                                double Qij, double Gi, double Gj, double C)
{
    const double TAU = 1e-12;
    if (yi != yj) {
        double quad = QDi + QDj + 2 * Qij;
        if (quad <= 0) quad = TAU;
        const double delta = (-Gi - Gj) / quad;
        const double diff = ai - aj;
        ai += delta;
        aj += delta;
        if (diff > 0) {
            if (aj < 0) {
                aj = 0;
                ai = diff;
            }
        } else {
            if (ai < 0) {
                ai = 0;
                aj = -diff;
            }
        }
        if (diff > C - C) {
            if (ai > C) {
                ai = C;
                aj = C - diff;
            }
        } else {
            if (aj > C) {
                aj = C;
                ai = C + diff;
            }
        }
    } else {
        double quad = QDi + QDj - 2 * Qij;
        if (quad <= 0) quad = TAU;
        const double delta = (Gi - Gj) / quad;
        const double sum = ai + aj;
        ai -= delta;
        aj += delta;
        if (sum > C) {
            if (ai > C) {
                ai = C;
                aj = sum - C;
            }
        } else {
            if (aj < 0) {
                aj = 0;
                ai = sum;
            }
        }
        if (sum > C) {
            if (aj > C) {
                aj = C;
                ai = sum - C;
            }
        } else {
            if (ai < 0) {
                ai = 0;
                aj = sum;
            }
        }
    }
}

// libsvm's calculate_rho over positions [0, cnt) (lane l holds positions l and l + 32): the bounds' min / max in any
// order, sum_free added sequentially in position order as libsvm's loop adds it; the same value on every lane
__device__ __forceinline__ double svm_rho(const double (&y)[2], const double (&G)[2], const double (&alpha)[2], int cnt,
                                          double C)
{
    const int lane = threadIdx.x & 31;
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    double ub = INF, lb = -INF, yG_free[2];
    int nr_free = 0;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        yG_free[s] = 0.0;
        if (lane + 32 * s >= cnt) continue;
        const double yG = y[s] * G[s];
        if (alpha[s] >= C) {
            if (y[s] < 0) ub = fmin(ub, yG); else lb = fmax(lb, yG);
        } else if (alpha[s] <= 0) {
            if (y[s] > 0) ub = fmin(ub, yG); else lb = fmax(lb, yG);
        } else {
            ++nr_free;
            yG_free[s] = yG;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        ub = fmin(ub, __shfl_xor_sync(0xffffffffu, ub, off));
        lb = fmax(lb, __shfl_xor_sync(0xffffffffu, lb, off));
        nr_free += __shfl_xor_sync(0xffffffffu, nr_free, off);
    }
    if (nr_free == 0) return (ub + lb) / 2;
    double sum_free = 0.0;   // + 0.0 for a bounded position leaves the sum unchanged (it is never -0)
    for (int k = 0; k < cnt; k++) sum_free = __dadd_rn(sum_free, warp_at(yG_free, k));
    return sum_free / nr_free;
}

// The held-out decisions as libsvm's svm_predict_values forms them: dec = sum_k (alpha_k y_k) K(t, k) - rho with the
// support vectors added sequentially in training order (class +1 first), each product and sum rounded on its own; dec > 0
// -> the first class.  coef[k] = alpha_k y_k by training index k (per-warp shared memory).  Lane l predicts held-out
// samples l and l + 32.  bits: bit t set when sample t falls on the first class's side; ok: correctly predicted samples.
template <typename KT>
__device__ __forceinline__ void svm_predict(const SvmFold &fd, const KT *__restrict__ Kp, int E, const double *coef,
                                            double rho, int &ok, unsigned long long &bits)
{
    const int lane = threadIdx.x & 31;
    bool pos[2], hit[2];
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const int t = lane + 32 * s;
        pos[s] = hit[s] = false;
        if (t >= fd.n_test) continue;
        const KT *row = Kp + (size_t)fd.test_idx[t] * E;
        double sum = 0.0;
        for (int k = 0; k < fd.n_train; k++) {
            const double c = coef[k];
            if (c != 0.0) sum = __dadd_rn(sum, __dmul_rn(c, (double)row[fd.train_idx[k]]));
        }
        pos[s] = __dsub_rn(sum, rho) > 0;
        hit[s] = pos[s] == (fd.test_pos[t] != 0);
    }
    bits = (unsigned long long)__ballot_sync(0xffffffffu, pos[0]) |
           ((unsigned long long)__ballot_sync(0xffffffffu, pos[1]) << 32);
    ok = __popc(__ballot_sync(0xffffffffu, hit[0])) + __popc(__ballot_sync(0xffffffffu, hit[1]));
}

// Kernel element type KT: float (the FCMA kernels) or double (searchlight kernels).  Either way Q is float and QD, the
// gradient and the decisions are double, as libsvm keeps them; an fp64 kernel therefore reproduces what libsvm computes
// for a non-precomputed kernel (QD and the decision values from the double kernel function).  The double form reads the
// decisions' kernel values from Kpred (the rbf difference form of k_function); the float form ignores Kpred.  Q is
// formed as y_a y_b (float)K, which equals (float)(y_a y_b K) because y_a y_b = +-1 and rounding commutes with the sign.
//
// SHRINK adds libsvm's shrinking heuristic (scikit-learn's default shrinking=True): Solver::do_shrinking, be_shrunk,
// reconstruct_gradient, swap_index and the counter / unshrink logic of Solver::Solve restated for one warp.  Lanes own
// POSITIONS lane and lane+32 of libsvm's permuted arrays; an item's state (y, alpha, G, G_bar, QD and its index `pm` in
// the unpermuted sub-problem = active_set[]) travels between positions through the warp's SvmStage when do_shrinking
// swaps; Q stays in the unpermuted order and is addressed through pm.  Working-set selection, the G update and rho run
// over [0, active); G_bar over all n.  Without SHRINK, active = n and every item stays at its own position.
template <typename KT, bool SHRINK>
__global__ void __launch_bounds__(128) k_svm_cv(const KT *__restrict__ K, long nv, int E, int nfolds,
                                               const SvmFold *__restrict__ folds, double C, double eps, int max_iter,
                                               int *__restrict__ correct, int *__restrict__ iters,
                                               unsigned long long *__restrict__ dec_bits, const KT *__restrict__ Kpred)
{
    extern __shared__ float s_q[];   // svm_smem_bytes(SHRINK): [4 warps][64][64] Q, then with SHRINK [4 warps] SvmStage
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long prob = (long)blockIdx.x * 4 + warp;
    if (prob >= nv * nfolds) return;
    const long v = prob / nfolds;
    const int f = (int)(prob - v * nfolds);
    const SvmFold &fd = folds[f];
    const int n = fd.n_train;
    const KT *Kv = K + (size_t)v * E * E;
    const KT *Kp = sizeof(KT) == 4 ? Kv : Kpred + (size_t)v * E * E;
    float *Q = s_q + (size_t)warp * 64 * 64;
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    const double TAU = 1e-12;
    const unsigned FULL = 0xffffffffu;

    // the item at a position: its index in the unpermuted sub-problem (Q's row / column) and its y, on every lane; and
    // the index of this lane's slot s.  Without shrinking that is the position itself and y follows from it.
    int pm[2];
    double y[2];
    auto index_at = [&](int pos) {
        if constexpr (SHRINK) return warp_at(pm, pos); else return pos;
    };
    auto own_index = [&](int s) {
        if constexpr (SHRINK) return pm[s]; else return lane + 32 * s;
    };
    auto y_at = [&](int pos) {
        if constexpr (SHRINK) return warp_at(y, pos); else return pos < fd.n_pos ? 1.0 : -1.0;
    };

    // sub-problem in libsvm's order; Q_ab = (float)(y_a y_b K_ab)
    int idx[2];
    double alpha[2], G[2], Gb[2], QD[2];
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const int k = lane + 32 * s;
        pm[s] = k < n ? k : 0;
        idx[s] = k < n ? fd.train_idx[k] : 0;
        y[s] = k < fd.n_pos ? 1.0 : -1.0;
        alpha[s] = 0.0;
        G[s] = -1.0;   // p = -1
        Gb[s] = 0.0;
    }
    for (int a = 0; a < n; a++) {
        const int ia = fd.train_idx[a];
        const float ya = a < fd.n_pos ? 1.f : -1.f;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k < n) Q[a * 64 + k] = ya * (float)y[s] * (float)Kv[(size_t)ia * E + idx[s]];
        }
    }
    __syncwarp();
#pragma unroll
    for (int s = 0; s < 2; s++) QD[s] = lane + 32 * s < n ? (double)Kv[(size_t)idx[s] * E + idx[s]] : 0.0;

    int active = n;
    bool unshrink = false;
    int counter = (n < 1000 ? n : 1000) + 1;

    // Solver::select_working_set (second order) over [0, active); true = already optimal (libsvm returns 1)
    auto select = [&](int &i, int &j) -> bool {
        double Gmax = -INF;
        i = -1;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= active) continue;
            double cand = -INF;
            if (y[s] > 0) {
                if (!(alpha[s] >= C)) cand = -G[s];
            } else {
                if (!(alpha[s] <= 0)) cand = G[s];
            }
            if (cand >= Gmax && cand > -INF) {
                Gmax = cand;
                i = k;
            }
        }
        warp_argbest(Gmax, i, true);
        j = -1;
        if (i < 0) return true;
        const double yi = y_at(i), QDi = warp_at(QD, i);
        const float *Qi = Q + index_at(i) * 64;
        double Gmax2 = -INF, obj_min = INF;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= active) continue;
            const double Qik = (double)Qi[own_index(s)];
            if (y[s] > 0) {
                if (!(alpha[s] <= 0)) {
                    const double gd = Gmax + G[s];
                    if (G[s] >= Gmax2) Gmax2 = G[s];
                    if (gd > 0) {
                        const double quad = QDi + QD[s] - 2.0 * yi * Qik;
                        const double obj = quad > 0 ? -(gd * gd) / quad : -(gd * gd) / TAU;
                        if (obj <= obj_min) {
                            j = k;
                            obj_min = obj;
                        }
                    }
                }
            } else {
                if (!(alpha[s] >= C)) {
                    const double gd = Gmax - G[s];
                    if (-G[s] >= Gmax2) Gmax2 = -G[s];
                    if (gd > 0) {
                        const double quad = QDi + QD[s] + 2.0 * yi * Qik;
                        const double obj = quad > 0 ? -(gd * gd) / quad : -(gd * gd) / TAU;
                        if (obj <= obj_min) {
                            j = k;
                            obj_min = obj;
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            double o = __shfl_xor_sync(FULL, Gmax2, off);
            Gmax2 = o > Gmax2 ? o : Gmax2;
        }
        warp_argbest(obj_min, j, false);
        return (Gmax + Gmax2 < eps) || j < 0;
    };

    // Solver::reconstruct_gradient: G of the inactive positions from G_bar and the free active variables (both of libsvm's
    // loop orders add the free variables in ascending position; they differ in which triangle of Q they read)
    auto reconstruct = [&]() {
        if (active == n) return;
        int nr_free = 0;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= active && k < n) G[s] = __dadd_rn(Gb[s], -1.0);
            if (k < active && !(alpha[s] >= C) && !(alpha[s] <= 0)) ++nr_free;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) nr_free += __shfl_xor_sync(FULL, nr_free, off);
        const bool by_rows = (long)nr_free * n > 2L * active * (n - active);
        for (int jj = 0; jj < active; jj++) {
            const double a_j = warp_at(alpha, jj);
            const int pm_j = warp_at(pm, jj);
            if (a_j >= C || a_j <= 0) continue;
#pragma unroll
            for (int s = 0; s < 2; s++) {
                const int k = lane + 32 * s;
                if (k >= active && k < n) {
                    const float q = by_rows ? Q[pm[s] * 64 + pm_j] : Q[pm_j * 64 + pm[s]];
                    G[s] = __dadd_rn(G[s], __dmul_rn(a_j, (double)q));
                }
            }
        }
    };

    // Solver::do_shrinking
    auto do_shrinking = [&]() {
        double g1 = -INF, g2 = -INF;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= active) continue;
            const bool up = alpha[s] >= C, low = alpha[s] <= 0;
            if (y[s] > 0) {
                if (!up && -G[s] >= g1) g1 = -G[s];
                if (!low && G[s] >= g2) g2 = G[s];
            } else {
                if (!up && -G[s] >= g2) g2 = -G[s];
                if (!low && G[s] >= g1) g1 = G[s];
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double o1 = __shfl_xor_sync(FULL, g1, off), o2 = __shfl_xor_sync(FULL, g2, off);
            g1 = o1 > g1 ? o1 : g1;
            g2 = o2 > g2 ? o2 : g2;
        }
        if (!unshrink && g1 + g2 <= eps * 10) {
            unshrink = true;
            reconstruct();
            active = n;
        }
        bool fl[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            fl[s] = false;
            if (k >= active) continue;
            if (alpha[s] >= C)
                fl[s] = y[s] > 0 ? (-G[s] > g1) : (-G[s] > g2);
            else if (alpha[s] <= 0)
                fl[s] = y[s] > 0 ? (G[s] > g2) : (G[s] > g1);
        }
        unsigned long long F = (unsigned long long)__ballot_sync(FULL, fl[0]) |
                               ((unsigned long long)__ballot_sync(FULL, fl[1]) << 32);
        if (F == 0ull) return;
        SvmStage &stg = reinterpret_cast<SvmStage *>(s_q + SVM_Q_FLOATS)[warp];
        stg.map[lane] = (unsigned char)lane;
        stg.map[lane + 32] = (unsigned char)(lane + 32);
        __syncwarp();
        int act = active, swaps = 0;
        if (lane == 0) {
            // the serial scan of libsvm (flags travel with the items: after swap_index(i, act) position i holds the
            // unflagged item and position act the flagged one)
            for (int i = 0; i < act; i++)
                if ((F >> i) & 1ull) {
                    act--;
                    while (act > i) {
                        if (!((F >> act) & 1ull)) {
                            const unsigned char t = stg.map[i];
                            stg.map[i] = stg.map[act];
                            stg.map[act] = t;
                            F ^= (1ull << i) | (1ull << act);
                            ++swaps;
                            break;
                        }
                        act--;
                    }
                }
        }
        act = __shfl_sync(FULL, act, 0);
        swaps = __shfl_sync(FULL, swaps, 0);
        active = act;
        if (swaps == 0) return;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            stg.d[0][k] = G[s];
            stg.d[1][k] = Gb[s];
            stg.d[2][k] = alpha[s];
            stg.d[3][k] = QD[s];
            stg.i[0][k] = pm[s];
            stg.i[1][k] = y[s] > 0 ? 1 : 0;
        }
        __syncwarp();
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= n) continue;
            const int src = stg.map[k];
            G[s] = stg.d[0][src];
            Gb[s] = stg.d[1][src];
            alpha[s] = stg.d[2][src];
            QD[s] = stg.d[3][src];
            pm[s] = stg.i[0][src];
            y[s] = stg.i[1][src] ? 1.0 : -1.0;
        }
        __syncwarp();
    };

    int iter = 0;
    while (true) {
        if (max_iter >= 0 && iter >= max_iter) break;
        int i, j;
        if constexpr (SHRINK) {
            if (--counter == 0) {
                counter = n < 1000 ? n : 1000;
                do_shrinking();
            }
            if (select(i, j)) {
                reconstruct();
                active = n;
                if (select(i, j)) break;
                counter = 1;   // do shrinking next iteration
            }
        } else if (select(i, j)) {
            break;
        }
        ++iter;

        // ---- analytic update of (alpha_i, alpha_j) with libsvm's clipping, then G (and G_bar) of every position
        const double yi = y_at(i), yj = y_at(j), QDi = warp_at(QD, i), QDj = warp_at(QD, j);
        const double Gi = warp_at(G, i), Gj = warp_at(G, j);
        const int pmi = index_at(i), pmj = index_at(j);
        const float *Qi = Q + pmi * 64, *Qj = Q + pmj * 64;
        double ai = warp_at(alpha, i), aj = warp_at(alpha, j);
        const double old_ai = ai, old_aj = aj;
        smo_pair_update(ai, aj, yi, yj, QDi, QDj, (double)Qi[pmj], Gi, Gj, C);
        const double dai = ai - old_ai, daj = aj - old_aj;
        const bool ui = old_ai >= C, uj = old_aj >= C, ui2 = ai >= C, uj2 = aj >= C;   // G_bar's bound changes
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int k = lane + 32 * s;
            if (k >= n) continue;
            const double qi = (double)Qi[own_index(s)], qj = (double)Qj[own_index(s)];
            // G[k] += Q_i[k]*dai + Q_j[k]*daj, no FMA contraction (as the reference compiles it)
            if (k < active) G[s] = __dadd_rn(G[s], __dadd_rn(__dmul_rn(qi, dai), __dmul_rn(qj, daj)));
            if constexpr (SHRINK) {
                if (ui != ui2) Gb[s] = ui ? __dsub_rn(Gb[s], __dmul_rn(C, qi)) : __dadd_rn(Gb[s], __dmul_rn(C, qi));
                if (uj != uj2) Gb[s] = uj ? __dsub_rn(Gb[s], __dmul_rn(C, qj)) : __dadd_rn(Gb[s], __dmul_rn(C, qj));
            }
            if (k == i) alpha[s] = ai;
            if (k == j) alpha[s] = aj;
        }
    }

    // ---- rho (calculate_rho over the active positions: all of them unless max_iter cut the loop)
    const double rho = svm_rho(y, G, alpha, active, C);

    // ---- predict the held-out samples in training order: Q is no longer read, its space stages alpha_k y_k by
    // unpermuted index
    double *coef = reinterpret_cast<double *>(Q);
    __syncwarp();
#pragma unroll
    for (int s = 0; s < 2; s++)
        if (lane + 32 * s < n) coef[own_index(s)] = alpha[s] * y[s];
    __syncwarp();
    int ok;
    unsigned long long bits;
    svm_predict(fd, Kp, E, coef, rho, ok, bits);
    if (lane == 0) {
        if (correct) correct[prob] = ok;
        if (iters) iters[prob] = iter;
        if (dec_bits) dec_bits[prob] = bits;
    }
}

extern "C" int fcma_shrink_kernels(float *K_dev, long nv, int E, int *digits_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!K_dev || nv <= 0 || E <= 0) return fail(FCMA_EINVAL, "fcma_shrink_kernels: bad arguments");
    k_shrink_kernels<<<(unsigned)cdiv(nv, 4), 128, 0, (cudaStream_t)stream>>>(K_dev, nv, E, digits_dev);
    LAUNCH_CHECK("k_shrink_kernels");
    return FCMA_OK;
}

template <typename KT>
static int svm_cv_impl(const KT *K_dev, const KT *Kpred_dev, long nv, int E, int nfolds, const void *folds_host, double C,
                       double tol, int max_iter, int shrinking, int *correct_dev, int *iters_dev,
                       unsigned long long *bits_dev, void *stream);
extern "C" int fcma_svm_cv_precomputed(const float *K_dev, long nv, int E, int nfolds, const void *folds_host,
                                       double C, double tol, int max_iter, int *correct_dev, int *iters_dev,
                                       void *stream)
{
    if (!correct_dev) return fail(FCMA_EINVAL, "fcma_svm_cv_precomputed: null output");
    return svm_cv_impl<float>(K_dev, nullptr, nv, E, nfolds, folds_host, C, tol, max_iter, 0, correct_dev, iters_dev,
                              nullptr, stream);
}
// the general form: `shrinking` selects the restatement of libsvm's shrinking heuristic (scikit-learn's default); bits_dev
// (optional) receives the binary DECISION of every held-out sample (bit t of bits_dev[v * nproblems + p]) -- the building
// block of one-vs-one multi-class cross-validation (one "fold" struct per (fold, class pair), votes on the caller's side)
extern "C" int fcma_svm_cv_solve(const float *K_dev, long nv, int E, int nproblems, const void *folds_host, double C,
                                 double tol, int max_iter, int shrinking, int *correct_dev,
                                 unsigned long long *bits_dev, int *iters_dev, void *stream)
{
    if (!bits_dev && !correct_dev) return fail(FCMA_EINVAL, "fcma_svm_cv_solve: no output requested");
    return svm_cv_impl<float>(K_dev, nullptr, nv, E, nproblems, folds_host, C, tol, max_iter, shrinking, correct_dev,
                              iters_dev, bits_dev, stream);
}
// the same solver on fp64 kernels: Q_ab = (float)(y_a y_b K_fit_ab), QD_a = K_fit_aa and the decisions
// sum_k alpha_k y_k K_pred[t][k] - rho in double.  K_pred may be K_fit (linear kernel).
extern "C" int fcma_svm_cv_solve_f64(const double *K_fit_dev, const double *K_pred_dev, long nv, int E, int nproblems,
                                     const void *folds_host, double C, double tol, int max_iter, int shrinking,
                                     int *correct_dev, unsigned long long *bits_dev, int *iters_dev, void *stream)
{
    if (!bits_dev && !correct_dev) return fail(FCMA_EINVAL, "fcma_svm_cv_solve_f64: no output requested");
    if (!K_pred_dev) return fail(FCMA_EINVAL, "fcma_svm_cv_solve_f64: null K_pred");
    return svm_cv_impl<double>(K_fit_dev, K_pred_dev, nv, E, nproblems, folds_host, C, tol, max_iter, shrinking,
                               correct_dev, iters_dev, bits_dev, stream);
}
template <typename KT>
static int svm_cv_impl(const KT *K_dev, const KT *Kpred_dev, long nv, int E, int nfolds, const void *folds_host, double C,
                       double tol, int max_iter, int shrinking, int *correct_dev, int *iters_dev,
                       unsigned long long *bits_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!K_dev || !folds_host || nv <= 0 || E <= 0 || E > 64 || nfolds <= 0 || nfolds > 4096)
        return fail(FCMA_EINVAL, "fcma_svm_cv_precomputed: bad arguments (E <= 64, at most 4096 fold problems)");
    if (!(C > 0) || !(tol > 0)) return fail(FCMA_EINVAL, "fcma_svm_cv_precomputed: C and tol must be positive");
    const SvmFold *fh = reinterpret_cast<const SvmFold *>(folds_host);
    for (int f = 0; f < nfolds; f++) {
        if (fh[f].n_train < 2 || fh[f].n_train > 64 || fh[f].n_test < 0 || fh[f].n_test > 64 || fh[f].n_pos < 1 ||
            fh[f].n_pos >= fh[f].n_train)
            return fail(FCMA_EINVAL, "fold %d: need both classes in the training part and <= 64 samples", f);
        for (int k = 0; k < fh[f].n_train; k++)
            if (fh[f].train_idx[k] < 0 || fh[f].train_idx[k] >= E) return fail(FCMA_EINVAL, "fold %d: bad train index", f);
        for (int k = 0; k < fh[f].n_test; k++)
            if (fh[f].test_idx[k] < 0 || fh[f].test_idx[k] >= E) return fail(FCMA_EINVAL, "fold %d: bad test index", f);
    }
    cudaStream_t st = (cudaStream_t)stream;
    AsyncBuf fd_buf;
    CUDA_TRY(fd_buf.alloc(sizeof(SvmFold) * nfolds, st));
    SvmFold *fd = static_cast<SvmFold *>(fd_buf.p);
    CUDA_TRY(cudaMemcpyAsync(fd, fh, sizeof(SvmFold) * nfolds, cudaMemcpyHostToDevice, st));
    return launch_kernel(shrinking ? k_svm_cv<KT, true> : k_svm_cv<KT, false>, (unsigned)cdiv(nv * nfolds, 4), 128,
                         svm_smem_bytes(shrinking), st, "k_svm_cv", K_dev, nv, E, nfolds, fd, C, tol, max_iter,
                         correct_dev, iters_dev, bits_dev, Kpred_dev);
}

// ============================================================================================
// Searchlight kernel matrices (MVPAVoxelSelector): for each centre c of a list, the [E][E] fp64 Gram matrix of the
// centre's features -- the voxels of its (2r+1)^3 cube where mask and shape both hold, in C order of the cube -- with
// the sample vectors x_e = vol[voxel][e] (volume [nx][ny][nz][E], epochs contiguous per voxel).
//   kind 0 (linear): K_fit = G,  G_ab = sum_f x_a[f] x_b[f]
//   kind 1 (rbf):    K_fit_ab  = exp(-gamma ((G_aa + G_bb) - 2 G_ab))   libsvm's kernel_rbf (x_square form, training)
//                    K_pred_ab = exp(-gamma sum_f (x_a[f] - x_b[f])^2)   libsvm's k_function (difference form, decisions)
// The products of float32 values are exact in fp64, so only the order of the additions (features in cube order, one
// sequential sum per pair) can differ from the reference's BLAS dot; every operation is rounded separately (no FMA
// contraction).  K_fit_aa is exactly 1 for rbf, as libsvm's QD.  One CTA per centre: the features' E-vectors are
// staged through shared memory in chunks of SL_CHUNK cube positions (any radius), each thread owns up to SL_PAIRS
// pairs a <= b of the upper triangle, and the finished matrix goes out through shared memory in coalesced rows.
#define SL_THREADS 256
#define SL_CHUNK 32
#define SL_PAIRS 9   // ceil(64 * 65 / 2 / SL_THREADS)

// libsvm's rbf kernel values from fp64 sums, each operation rounded separately: the x_square form its training uses
// (from the Gram entries G_aa, G_bb, G_ab; exactly 1 on the diagonal) and the difference form of its decisions (from
// d = sum_f (x_a - x_b)^2).  Shared by k_searchlight_kernels and k_norm_gram_f64.
__device__ __forceinline__ double rbf_fit(double gamma, double gaa, double gbb, double gab)
{
    return exp(__dmul_rn(-gamma, __dsub_rn(__dadd_rn(gaa, gbb), __dmul_rn(2.0, gab))));
}
__device__ __forceinline__ double rbf_pred(double gamma, double d) { return exp(__dmul_rn(-gamma, d)); }

template <int KIND>
__global__ void __launch_bounds__(SL_THREADS) k_searchlight_kernels(const float *__restrict__ vol, int ny, int nz, int E,
                                                                    const unsigned char *__restrict__ mask, int r,
                                                                    const unsigned char *__restrict__ shape,
                                                                    const long *__restrict__ centres,
                                                                    const double *__restrict__ gamma,
                                                                    double *__restrict__ K_fit, double *__restrict__ K_pred)
{
    extern __shared__ double s_sl[];
    double *tile = s_sl;                                                   // [E][E]
    double *diag = tile + E * E;                                           // [E] G_aa
    float *xs = reinterpret_cast<float *>(diag + E);                       // [SL_CHUNK][E]
    unsigned char *act = reinterpret_cast<unsigned char *>(xs + SL_CHUNK * E);   // [SL_CHUNK]
    const int tid = threadIdx.x;
    const long m = blockIdx.x;
    const long c = centres[m];
    const int cz = (int)(c % nz), cy = (int)((c / nz) % ny), cx = (int)(c / ((long)nz * ny));
    const int side = 2 * r + 1, ncube = side * side * side;
    const int P = E * (E + 1) / 2;

    int pa[SL_PAIRS], pb[SL_PAIRS];
    double g[SL_PAIRS], d[SL_PAIRS];
#pragma unroll
    for (int s = 0; s < SL_PAIRS; s++) {
        const int p = tid + s * SL_THREADS;
        int a = 0, rem = p;
        // row a of the upper triangle holds the E - a pairs (a, a..E-1)
        while (p < P && rem >= E - a) rem -= E - a++;
        pa[s] = p < P ? a : -1;
        pb[s] = p < P ? a + rem : -1;
        g[s] = 0.0;
        d[s] = 0.0;
    }

    for (int o0 = 0; o0 < ncube; o0 += SL_CHUNK) {
        const int nch = min(SL_CHUNK, ncube - o0);
        __syncthreads();
        if (tid < nch) {
            const int o = o0 + tid;
            const int i = o / (side * side), j = (o / side) % side, k = o % side;
            const long vox = ((long)(cx - r + i) * ny + (cy - r + j)) * nz + (cz - r + k);
            act[tid] = shape[o] && mask[vox];
        }
        __syncthreads();
        for (int idx = tid; idx < nch * E; idx += SL_THREADS) {
            const int q = idx / E, e = idx - q * E;
            if (act[q]) {
                const int o = o0 + q;
                const int i = o / (side * side), j = (o / side) % side, k = o % side;
                const long vox = ((long)(cx - r + i) * ny + (cy - r + j)) * nz + (cz - r + k);
                xs[q * E + e] = vol[vox * E + e];
            }
        }
        __syncthreads();
        for (int q = 0; q < nch; q++) {
            if (!act[q]) continue;
            const float *xq = xs + q * E;
#pragma unroll
            for (int s = 0; s < SL_PAIRS; s++) {
                if (pa[s] < 0) continue;
                const double xa = (double)xq[pa[s]], xb = (double)xq[pb[s]];
                g[s] = __dadd_rn(g[s], __dmul_rn(xa, xb));
                if (KIND == 1) {
                    const double df = __dsub_rn(xa, xb);
                    d[s] = __dadd_rn(d[s], __dmul_rn(df, df));
                }
            }
        }
    }

    const size_t base = (size_t)m * E * E;
    if (KIND == 1) {
#pragma unroll
        for (int s = 0; s < SL_PAIRS; s++)
            if (pa[s] >= 0 && pa[s] == pb[s]) diag[pa[s]] = g[s];
    }
    __syncthreads();
    const double gm = KIND == 1 ? gamma[m] : 0.0;
#pragma unroll
    for (int s = 0; s < SL_PAIRS; s++) {
        if (pa[s] < 0) continue;
        double v = g[s];
        if (KIND == 1) v = rbf_fit(gm, diag[pa[s]], diag[pb[s]], g[s]);
        tile[pa[s] * E + pb[s]] = v;
        tile[pb[s] * E + pa[s]] = v;
    }
    __syncthreads();
    for (int idx = tid; idx < E * E; idx += SL_THREADS) K_fit[base + idx] = tile[idx];
    if (KIND == 1) {
        __syncthreads();
#pragma unroll
        for (int s = 0; s < SL_PAIRS; s++) {
            if (pa[s] < 0) continue;
            const double v = rbf_pred(gm, d[s]);
            tile[pa[s] * E + pb[s]] = v;
            tile[pb[s] * E + pa[s]] = v;
        }
        __syncthreads();
        for (int idx = tid; idx < E * E; idx += SL_THREADS) K_pred[base + idx] = tile[idx];
    }
}

extern "C" int fcma_searchlight_kernels(const float *vol_dev, long nx, long ny, long nz, int E,
                                        const unsigned char *mask_dev, int sl_rad, const unsigned char *shape_dev,
                                        const long *centres_host, long M, int kind, const double *gamma_host,
                                        double *K_fit_dev, double *K_pred_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (!vol_dev || !mask_dev || !shape_dev || !centres_host || !K_fit_dev || M <= 0 || nx <= 0 || ny <= 0 || nz <= 0)
        return fail(FCMA_EINVAL, "fcma_searchlight_kernels: null buffer or empty volume / centre list");
    if (E < 1 || E > 64) return fail(FCMA_EINVAL, "fcma_searchlight_kernels: E = %d outside 1..64", E);
    if (sl_rad < 0) return fail(FCMA_EINVAL, "fcma_searchlight_kernels: negative sl_rad");
    if (kind != 0 && kind != 1) return fail(FCMA_EINVAL, "fcma_searchlight_kernels: kind must be 0 (linear) or 1 (rbf)");
    if (kind == 1 && (!gamma_host || !K_pred_dev))
        return fail(FCMA_EINVAL, "fcma_searchlight_kernels: rbf needs gamma and K_pred");
    if (M > 0x7fffffffL) return fail(FCMA_EINVAL, "fcma_searchlight_kernels: too many centres in one call");
    for (long m = 0; m < M; m++) {
        const long c = centres_host[m];
        if (c < 0 || c >= nx * ny * nz) return fail(FCMA_EINVAL, "centre %ld: index %ld outside the volume", m, c);
        const long z = c % nz, y = (c / nz) % ny, x = c / (nz * ny);
        if (x < sl_rad || y < sl_rad || z < sl_rad || x >= nx - sl_rad || y >= ny - sl_rad || z >= nz - sl_rad)
            return fail(FCMA_EINVAL, "centre %ld (%ld, %ld, %ld) is closer than sl_rad = %d to a face", m, x, y, z, sl_rad);
    }
    cudaStream_t st = (cudaStream_t)stream;
    AsyncBuf cbuf, gbuf;
    CUDA_TRY(cbuf.alloc(sizeof(long) * M, st));
    CUDA_TRY(cudaMemcpyAsync(cbuf.p, centres_host, sizeof(long) * M, cudaMemcpyHostToDevice, st));
    if (kind == 1) {
        CUDA_TRY(gbuf.alloc(sizeof(double) * M, st));
        CUDA_TRY(cudaMemcpyAsync(gbuf.p, gamma_host, sizeof(double) * M, cudaMemcpyHostToDevice, st));
    }
    const size_t smem = (size_t)E * E * sizeof(double) + E * sizeof(double) + SL_CHUNK * E * sizeof(float) + SL_CHUNK;
    const long *cdev = static_cast<const long *>(cbuf.p);
    const double *gdev = static_cast<const double *>(gbuf.p);
    if (kind == 0)
        return launch_kernel(k_searchlight_kernels<0>, (unsigned)M, SL_THREADS, smem, st, "k_searchlight_kernels",
                             vol_dev, (int)ny, (int)nz, E, mask_dev, sl_rad, shape_dev, cdev, gdev, K_fit_dev,
                             K_pred_dev);
    return launch_kernel(k_searchlight_kernels<1>, (unsigned)M, SL_THREADS, smem, st, "k_searchlight_kernels", vol_dev,
                         (int)ny, (int)nz, E, mask_dev, sl_rad, shape_dev, cdev, gdev, K_fit_dev, K_pred_dev);
}

// ============================================================================================
// Per-voxel fp64 kernel matrices of the normalised correlation vectors (VoxelSelector with SVC(kernel='linear' | 'rbf')):
// for voxel row i of a raw correlation block, z = within_subject_column(r) (bit-identical to k_within_subject_norm), then
//   G_ab = sum_j z_aj z_bj          on the fp64 tensor cores (mma.sync m8n8k4 f64; fp32 products are exact in fp64)
//   D_ab = sum_j (z_aj - z_bj)^2    rbf only, on the FP64 pipe (difference in fp64, then one fma)
// and the epilogue: linear K_fit = G; rbf K_fit = rbf_fit(G), K_pred = rbf_pred(D).  These are the kernel values libsvm
// computes for SVC(kernel=...) on the float32 features z, up to the order of the sums (DESIGN.md §3.8).
//
// One CTA per row (grid-stride).  The row's E x V2 block streams through shared memory in chunks of NG_CH columns: loaded
// one chunk ahead into registers, normalised in place as fp32 [E][NG_RSP], widened to fp64 transposed [NG_CH][EP + 4]
// (EP = E rounded up to 16, zero rows past E; the pad makes both the MMA fragments and the D rows conflict-free).
// G: the NB8 = EP/8 row blocks of 8 give NB8(NB8+1)/2 upper 8x8 tiles; warp w takes the tile rows p and NB8-1-p
// (p = w % (NB8/2): NB8+1 tiles, the same for every warp) over every WK-th k-step (WK = 16/NB8 k-groups), and the k-groups'
// partial tiles are added in k-group order at the end of the row.  D: thread q < 136 owns the entries (ty + 16u, tx + 16v),
// ty <= tx, of a 16 x 16 grid, each summed sequentially over j.  No atomics: two runs are bit-identical.
#define NG_THREADS 256
#define NG_CH 64        // columns per chunk; divides the 256-column tiles of the tiled block
#define NG_RSP 72       // fp32 row pitch of the chunk (conflict-free in both the normalisation and the widening)

__device__ __forceinline__ void dmma_m8n8k4(double (&d)[2], double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

// E > 32: 36 G tiles + 16 D sums per thread do not fit the 128 registers of two CTAs per SM without spills
template <int EP, int KIND>
__global__ void __launch_bounds__(NG_THREADS, EP == 64 ? 1 : 2)
    k_norm_gram_f64(const float *__restrict__ C, long nb, int E, long n2, long stride_i, long ld, long chunk_step, long t256,
                    int eps, double gamma, double *__restrict__ K_fit, double *__restrict__ K_pred)
{
    constexpr int NB8 = EP / 8, NP = NB8 / 2, WK = 8 / NP, RPT = EP / 16, LDT = EP + 4, NPF = EP / 16;
    extern __shared__ double s_ng[];
    double *zt = s_ng;                                             // [NG_CH][LDT] z (fp64), then the [EP][EP] result tile
    float *rs = reinterpret_cast<float *>(zt + NG_CH * LDT);       // [E][NG_RSP] the chunk of r, normalised in place
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int p = warp % NP, kq = warp / NP;
    const long nsubj = E / eps;
    int ty = 0, tx = 0;
    const bool dq = KIND == 1 && tid < 136;
    if (dq) {
        int q = tid;
        while (q >= 16 - ty) q -= 16 - ty++;
        tx = ty + q;
    }
    for (long i = blockIdx.x; i < nb; i += gridDim.x) {
        const float *Ci = C + (chunk_step != 256 ? (i / 256) * t256 * chunk_step + (i % 256) * stride_i : i * stride_i);
        float4 pf[NPF];
        auto prefetch = [&](long j0) {
            const float *src = Ci + (j0 / 256) * chunk_step + j0 % 256;
#pragma unroll
            for (int k = 0; k < NPF; k++) {
                const int idx = tid + k * NG_THREADS, e = idx / (NG_CH / 4), c4 = idx % (NG_CH / 4);
                pf[k] = (e < E && j0 + 4 * c4 < n2) ? __ldg(reinterpret_cast<const float4 *>(src + e * ld + 4 * c4))
                                                    : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        };
        double acc[NB8 + 1][2];
        double dacc[RPT][RPT];
#pragma unroll
        for (int u = 0; u <= NB8; u++) acc[u][0] = acc[u][1] = 0.0;
#pragma unroll
        for (int a = 0; a < RPT; a++)
#pragma unroll
            for (int b = 0; b < RPT; b++) dacc[a][b] = 0.0;
        prefetch(0);
        for (long j0 = 0; j0 < n2; j0 += NG_CH) {
            __syncthreads();   // the previous chunk (and the previous row's result tile) is consumed
#pragma unroll
            for (int k = 0; k < NPF; k++) {
                const int idx = tid + k * NG_THREADS, e = idx / (NG_CH / 4), c4 = idx % (NG_CH / 4);
                float4 v = pf[k];
                // columns past n2 (inside the last float4, or pad of the block) are zero: they add nothing to G or D
                const long j = j0 + 4 * c4;
                if (j + 1 >= n2) v.y = 0.f;
                if (j + 2 >= n2) v.z = 0.f;
                if (j + 3 >= n2) v.w = 0.f;
                if (e < E) *reinterpret_cast<float4 *>(rs + e * NG_RSP + 4 * c4) = v;
            }
            if (j0 + NG_CH < n2) prefetch(j0 + NG_CH);
            __syncthreads();
            // epochs past the last whole subject keep their raw r, as in k_within_subject_norm
            for (int idx = tid; idx < nsubj * NG_CH; idx += NG_THREADS)
                within_subject_column(rs + idx % NG_CH, NG_RSP, idx / NG_CH, eps);
            __syncthreads();
            for (int idx = tid; idx < EP * NG_CH; idx += NG_THREADS) {
                const int grp = idx >> 5, l = idx & 31;
                const int e = (grp % (EP / 4)) * 4 + (l & 3), c = (grp / (EP / 4)) * 8 + (l >> 2);
                zt[c * LDT + e] = e < E ? (double)rs[e * NG_RSP + c] : 0.0;
            }
            __syncthreads();
            for (int ks = kq; ks < NG_CH / 4; ks += WK) {
                const double *zk = zt + (ks * 4 + t) * LDT + g;
                const double fa = zk[p * 8], fb = zk[(NB8 - 1 - p) * 8];
#pragma unroll
                for (int u = 0; u <= NB8; u++) {
                    // tiles (p, p..NB8-1), then (NB8-1-p, NB8-1-p..NB8-1)
                    const bool first = u < NB8 - p;
                    dmma_m8n8k4(acc[u], first ? fa : fb, zk[(first ? p + u : u - 1) * 8]);
                }
            }
            if (dq) {
                for (int c = 0; c < NG_CH; c++) {
                    const double *zc = zt + c * LDT;
                    double za[RPT], zb[RPT];
#pragma unroll
                    for (int u = 0; u < RPT; u++) za[u] = zc[ty + 16 * u], zb[u] = zc[tx + 16 * u];
#pragma unroll
                    for (int a = 0; a < RPT; a++)
#pragma unroll
                        for (int b = 0; b < RPT; b++) {
                            const double df = __dsub_rn(za[a], zb[b]);
                            dacc[a][b] = __fma_rn(df, df, dacc[a][b]);
                        }
                }
            }
        }
        // epilogue: G into the [EP][EP] tile (upper 8x8 tiles only), k-groups added in order
        double *tile = zt;
        for (int r = 0; r < WK; r++) {
            __syncthreads();
            if (kq == r) {
#pragma unroll
                for (int u = 0; u <= NB8; u++) {
                    const bool first = u < NB8 - p;
                    const int rb = first ? p : NB8 - 1 - p, cb = first ? p + u : u - 1;
                    double *dst = tile + (rb * 8 + g) * EP + cb * 8 + 2 * t;
                    dst[0] = r == 0 ? acc[u][0] : __dadd_rn(dst[0], acc[u][0]);
                    dst[1] = r == 0 ? acc[u][1] : __dadd_rn(dst[1], acc[u][1]);
                }
            }
        }
        __syncthreads();
        const size_t base = (size_t)i * E * E;
        for (int idx = tid; idx < E * E; idx += NG_THREADS) {
            const int a = idx / E, b = idx - a * E;
            double v = tile[min(a, b) * EP + max(a, b)];
            if (KIND == 1) v = rbf_fit(gamma, tile[a * EP + a], tile[b * EP + b], v);
            K_fit[base + idx] = v;
        }
        if (KIND == 1) {
            __syncthreads();
            if (dq) {
#pragma unroll
                for (int a = 0; a < RPT; a++)
#pragma unroll
                    for (int b = 0; b < RPT; b++) {
                        tile[(ty + 16 * a) * EP + tx + 16 * b] = dacc[a][b];
                        tile[(tx + 16 * b) * EP + ty + 16 * a] = dacc[a][b];
                    }
            }
            __syncthreads();
            for (int idx = tid; idx < E * E; idx += NG_THREADS) {
                const int a = idx / E, b = idx - a * E;
                K_pred[base + idx] = rbf_pred(gamma, tile[a * EP + b]);
            }
        }
    }
}

// (stride_i, ld, chunk_step, t256) address the raw correlation block as launch_norm_syrk's do (tiled: chunk_step = E*65536)
static int launch_norm_gram_f64(const float *C, long nb, int E, long n2, long stride_i, long ld, long chunk_step, long t256,
                                int eps, int kind, double gamma, double *K_fit, double *K_pred, cudaStream_t st)
{
    if (E < 1 || E > 64 || eps < 1) return fail(FCMA_EINVAL, "internal: k_norm_gram_f64 needs 1 <= E <= 64, eps >= 1");
    if (((uintptr_t)C & 15) || (ld & 3) || (stride_i & 3)) return fail(FCMA_EINVAL, "internal: k_norm_gram_f64 needs 16-byte rows");
    const long grid = nb < 16L * g_sm_count ? nb : 16L * g_sm_count;
    bool ok = false;
    int rc = FCMA_OK;
    auto go = [&](auto EP, auto KIND) {
        constexpr size_t smem = (size_t)NG_CH * (EP + 4) * sizeof(double) + (size_t)EP * NG_RSP * sizeof(float);
        rc = launch_kernel(k_norm_gram_f64<EP, KIND>, (unsigned)grid, NG_THREADS, smem, st, "k_norm_gram_f64", C, nb, E, n2,
                           stride_i, ld, chunk_step, t256, eps, gamma, K_fit, K_pred);
        ok = true;
    };
    auto per_kind = [&](auto EP) {
        if (kind == 0) go(EP, IntC<0>{});
        else go(EP, IntC<1>{});
    };
    if (E <= 16) per_kind(IntC<16>{});
    else if (E <= 32) per_kind(IntC<32>{});
    else per_kind(IntC<64>{});
    return ok ? rc : fail(FCMA_EINVAL, "internal: no k_norm_gram_f64 instantiation for E=%d", E);
}

extern "C" int fcma_voxel_feature_kernels(const void *rows_op, const void *cols_op, int precision, int E, int T, long V,
                                          long V2, long start, long nb, int eps, int kind, double gamma, float *work_dev,
                                          size_t work_bytes, double *K_fit_dev, double *K_pred_dev, void *stream)
{
    int rc = check_device();
    if (rc) return rc;
    if (eps <= 0) return fail(FCMA_EINVAL, "fcma_voxel_feature_kernels: epochs_per_subj must be positive");
    if (E < 1 || E > 64) return fail(FCMA_EINVAL, "fcma_voxel_feature_kernels: E = %d outside 1..64", E);
    if (kind != 0 && kind != 1) return fail(FCMA_EINVAL, "fcma_voxel_feature_kernels: kind must be 0 (linear) or 1 (rbf)");
    if (!K_fit_dev || (kind == 1 && !K_pred_dev)) return fail(FCMA_EINVAL, "fcma_voxel_feature_kernels: null output");
    if (kind == 1 && !(gamma >= 0.0 && gamma <= 1.7976931348623157e308))
        return fail(FCMA_EINVAL, "fcma_voxel_feature_kernels: gamma must be finite and non-negative");
    FeatureStage fs{kind, gamma, K_fit_dev, K_pred_dev};
    return run_pipeline(rows_op, cols_op, precision, E, T, V, V2, start, nb, eps, 0, work_dev, work_bytes, nullptr, 0,
                        (cudaStream_t)stream, &fs);
}

// ---------------------------------------------------------------- host-buffer entry points
struct DevBuf {
    void *p = nullptr;
    ~DevBuf()
    {
        if (p) cudaFree(p);
    }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, n ? n : 1); }
};

extern "C" int fcma_host_voxel_kernels(const float *const *raw_host, const float *const *raw2_host, const int *T_e, int E,
                                       long V, long V2, long start, long nb, int eps, int precision, int normalize,
                                       int flags, int device, float *K_host)
{
    if (!raw_host || !T_e || !K_host || E <= 0 || V <= 0 || nb <= 0) return fail(FCMA_EINVAL, "fcma_host_voxel_kernels: bad arguments");
    if (fcma_device_count() == 0) return fail(FCMA_ENODEV, "no sm_90 device");
    DeviceGuard guard;   // the caller's current device is restored on every return path
    CUDA_TRY(cudaSetDevice(device));
    int rc = check_device();
    if (rc) return rc;
    int T = 0;
    for (int e = 0; e < E; e++) {
        if (T_e[e] <= 0) return fail(FCMA_EINVAL, "epoch %d has non-positive length", e);
        if (T_e[e] > T) T = T_e[e];
    }
    const bool two = raw2_host != nullptr;
    if (!two) V2 = V;
    cudaStream_t st = 0;
    DevBuf epochs, epochs2, opR, opC, work, K;
    // stage the epochs as [E][T][V] (zero rows beyond T_e)
    auto upload = [&](DevBuf &buf, const float *const *src, long W) -> int {
        size_t bytes = (size_t)E * T * W * sizeof(float);
        CUDA_TRY(buf.alloc(bytes));
        CUDA_TRY(cudaMemsetAsync(buf.p, 0, bytes, st));
        for (int e = 0; e < E; e++)
            CUDA_TRY(cudaMemcpyAsync((float *)buf.p + (size_t)e * T * W, src[e], (size_t)T_e[e] * W * sizeof(float),
                                     cudaMemcpyHostToDevice, st));
        return FCMA_OK;
    };
    rc = upload(epochs, raw_host, V);
    if (rc) return rc;
    size_t opb = fcma_operand_bytes(precision, E, T, V);
    if (!opb) return fail(FCMA_EINVAL, "unknown precision %d", precision);
    CUDA_TRY(opR.alloc(opb));
    rc = fcma_pack_operand((const float *)epochs.p, E, T, V, V, T_e, normalize, precision, opR.p, opb, st);
    if (rc) return rc;
    const void *colsp = opR.p;
    if (two) {
        rc = upload(epochs2, raw2_host, V2);
        if (rc) return rc;
        size_t opb2 = fcma_operand_bytes(precision, E, T, V2);
        CUDA_TRY(opC.alloc(opb2));
        rc = fcma_pack_operand((const float *)epochs2.p, E, T, V2, V2, T_e, normalize, precision, opC.p, opb2, st);
        if (rc) return rc;
        colsp = opC.p;
    }
    size_t per_row = fcma_work_bytes_per_row(E, V2);
    size_t freeb = 0, totalb = 0;
    CUDA_TRY(cudaMemGetInfo(&freeb, &totalb));
    long rows = (long)((freeb / 2) / per_row);
    if (rows > nb) rows = nb;
    if (rows > 4096) rows = 4096;
    if (rows < 1) return fail(FCMA_ENOMEM, "not enough device memory for one correlation row block");
    CUDA_TRY(work.alloc(per_row * rows));
    CUDA_TRY(K.alloc((size_t)nb * E * E * sizeof(float)));
    rc = fcma_voxel_kernels(opR.p, colsp, precision, E, T, V, V2, start, nb, eps, flags, (float *)work.p, per_row * rows,
                            (float *)K.p, st);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(K_host, K.p, (size_t)nb * E * E * sizeof(float), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return FCMA_OK;
}

// Single-mask worker loop from HOST buffers (what a ctypes / cgo binding of the reference's VoxelSelector would call when
// raw_data2 is None): H2D of the E epochs, packing, fcma_voxel_kernels_sym over all V rows, D2H of the [V][E][E] kernels,
// synchronously on `device`.  The copies overlap the kernels where the data flow allows it: the epochs go up in four
// groups and the first pass' GEMM follows group by group; the kernels of a pass are read back while the next pass runs.
// Device buffers come from the device's default stream-ordered pool, whose release threshold is raised once so that
// repeated calls reuse the memory instead of going back to the OS.
struct HostSymCtx {
    const float *epochs;
    int E, T;
    long V;
    const int *T_e;          // nullptr unless ragged
    int normalize, precision;
    void *op;
    size_t opb;
    const int *e0, *cnt;
    cudaEvent_t *landed;     // per group: its epochs are in HBM (recorded on the upload stream)
};
static int host_sym_prepare(void *vctx, int g, cudaStream_t st)
{
    HostSymCtx *c = static_cast<HostSymCtx *>(vctx);
    CUDA_TRY(cudaStreamWaitEvent(st, c->landed[g], 0));
    return pack_operand_impl(c->epochs, c->E, c->T, c->V, c->V, c->T_e, c->normalize, c->precision, 0, c->V, c->e0[g],
                             c->cnt[g], c->op, c->opb, st);
}

extern "C" int fcma_host_voxel_kernels_sym(const float *const *raw_host, const int *T_e, int E, long V, int eps,
                                           int precision, int normalize, int flags, int device, long rows_per_pass,
                                           float *K_host)
{
    if (!raw_host || !T_e || !K_host || E <= 0 || V <= 0) return fail(FCMA_EINVAL, "fcma_host_voxel_kernels_sym: bad arguments");
    if (fcma_device_count() == 0) return fail(FCMA_ENODEV, "no sm_90 device");
    DeviceGuard guard;
    CUDA_TRY(cudaSetDevice(device));
    int rc = check_device();
    if (rc) return rc;
    int T = 0;
    for (int e = 0; e < E; e++) {
        if (T_e[e] <= 0) return fail(FCMA_EINVAL, "epoch %d has non-positive length", e);
        if (T_e[e] > T) T = T_e[e];
    }
    static std::once_flag pool_once[64];
    if (device >= 0 && device < 64)
        std::call_once(pool_once[device], [&] {
            cudaMemPool_t pool;
            if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
                uint64_t keep = UINT64_MAX;
                cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
            }
            cudaGetLastError();
        });
    // two private streams: uploads / read-backs run beside the kernels (pinned host buffers make them asynchronous DMA)
    struct Streams {
        cudaStream_t main = nullptr, copy = nullptr;
        ~Streams()
        {
            if (main) cudaStreamDestroy(main);
            if (copy) cudaStreamDestroy(copy);
        }
    } ss;
    CUDA_TRY(cudaStreamCreateWithFlags(&ss.main, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&ss.copy, cudaStreamNonBlocking));
    cudaStream_t st = ss.main;
    const size_t opb = fcma_operand_bytes(precision, E, T, V);
    if (!opb) return fail(FCMA_EINVAL, "unknown precision %d", precision);
    const size_t ep_bytes = (size_t)E * T * V * sizeof(float), k_bytes = (size_t)V * E * E * sizeof(float);
    const size_t per_row = sym_row_bytes(precision, E, eps, flags, V, 0);
    size_t freeb = 0, totalb = 0;
    CUDA_TRY(cudaMemGetInfo(&freeb, &totalb));
    {
        // buffers of a previous call are cached in the pool: reusable, although cudaMemGetInfo counts them as used
        cudaMemPool_t pool;
        uint64_t reserved = 0, used = 0;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess &&
            cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved) == cudaSuccess &&
            cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) == cudaSuccess && reserved > used)
            freeb += (size_t)(reserved - used);
        cudaGetLastError();
    }
    long rows = rows_per_pass > 0 ? rows_per_pass : 4096;
    const size_t fixed = ep_bytes + opb + k_bytes + ((size_t)1 << 30);
    const long fit = freeb > fixed ? (long)((freeb - fixed) / per_row) : 0;
    if (rows > fit) rows = fit;
    if (rows > round_up(V, 256)) rows = round_up(V, 256);
    rows = rows / 256 * 256;
    if (rows < 256) return fail(FCMA_ENOMEM, "not enough device memory for a 256-row correlation block (%zu bytes per row)", per_row);
    // a second block lets the GEMMs of the first TWO passes follow the upload (more of the copy hidden)
    const bool two_blocks = fit >= 2 * rows && rows < round_up(V, 256);
    const size_t work_bytes_total = per_row * rows * (two_blocks ? 2 : 1);
    int rc_run = FCMA_OK;
    {
        AsyncBuf epochs, op, work, K;       // released in stream order on `st` when this scope ends
        CUDA_TRY(epochs.alloc(ep_bytes, st));
        CUDA_TRY(op.alloc(opb, st));
        CUDA_TRY(work.alloc(work_bytes_total, st));
        CUDA_TRY(K.alloc(k_bytes, st));
        CUDA_TRY(cudaMemsetAsync(K.p, 0, k_bytes, st));
        bool ragged = false;
        for (int e = 0; e < E; e++) ragged = ragged || T_e[e] != T;
        if (ragged) CUDA_TRY(cudaMemsetAsync(epochs.p, 0, ep_bytes, st));
        // upload in up to 4 epoch groups on the copy stream; the first pass' GEMM follows group by group
        EventSet<1> alloc_done;
        CUDA_TRY(alloc_done.create());
        CUDA_TRY(cudaEventRecord(alloc_done.ev[0], st));
        CUDA_TRY(cudaStreamWaitEvent(ss.copy, alloc_done.ev[0], 0));
        constexpr int MAXG = 4;
        const int ng = E >= MAXG ? MAXG : 1;
        int e0[MAXG], cnt[MAXG];
        EventSet<MAXG> landed;
        CUDA_TRY(landed.create());
        for (int gi = 0, e = 0; gi < ng; gi++) {
            e0[gi] = e;
            cnt[gi] = (E - e) / (ng - gi);
            for (int k = 0; k < cnt[gi]; k++, e++)
                CUDA_TRY(cudaMemcpyAsync((float *)epochs.p + (size_t)e * T * V, raw_host[e], (size_t)T_e[e] * V * sizeof(float),
                                         cudaMemcpyHostToDevice, ss.copy));
            CUDA_TRY(cudaEventRecord(landed.ev[gi], ss.copy));
        }
        HostSymCtx ctx{(const float *)epochs.p, E, T, V, ragged ? T_e : nullptr, normalize, precision, op.p, opb, e0, cnt, landed.ev};
        SymHostHooks hooks;
        hooks.ngroups = ng, hooks.e0 = e0, hooks.cnt = cnt, hooks.prepare = host_sym_prepare, hooks.ctx = &ctx;
        hooks.copy = ss.copy, hooks.K_host = K_host, hooks.two_buffers = two_blocks;
        rc_run = run_pipeline_sym(op.p, precision, E, T, V, 0, V, eps, flags, (float *)work.p, work_bytes_total, (float *)K.p, st, &hooks);
        // everything enqueued so far must finish before the buffers go back to the pool and the function returns
        cudaError_t e1 = cudaStreamSynchronize(st), e2 = cudaStreamSynchronize(ss.copy);
        if (!rc_run && (e1 != cudaSuccess || e2 != cudaSuccess))
            rc_run = fail(FCMA_ECUDA, "fcma_host_voxel_kernels_sym: %s", cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
    }
    if (rc_run) return rc_run;
    CUDA_TRY(cudaStreamSynchronize(st));      // the stream-ordered frees
    return FCMA_OK;
}

// ---------------------------------------------------------------- inter-process peer copies (one process per GPU)
// Copy-engine exchange of the epoch shards between the ranks of one box (the replacement of the reference's per-epoch
// comm.bcast loop, preprocessing.py:211-223, that does not occupy SMs the persistent GEMM needs): a rank exports the
// allocation behind a device pointer as a 64-byte CUDA IPC handle, the peers map it and cudaMemcpyAsync into / out of
// it over NVLink.  The library keeps no state: the caller owns handles, mappings and streams.
typedef CUresult (*PFN_cuMemGetAddressRange)(CUdeviceptr *, size_t *, CUdeviceptr);
extern "C" int fcma_ipc_get_handle(const void *dev_ptr, void *handle64, size_t *offset)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    if (!dev_ptr || !handle64 || !offset) return fail(FCMA_EINVAL, "fcma_ipc_get_handle: null pointer");
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    CUDA_TRY(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !fn) return fail(FCMA_ECUDA, "cuMemGetAddressRange entry point not available");
    CUdeviceptr base = 0;
    size_t size = 0;
    CUresult r = reinterpret_cast<PFN_cuMemGetAddressRange>(fn)(&base, &size, (CUdeviceptr)dev_ptr);
    if (r != CUDA_SUCCESS) return fail(FCMA_ECUDA, "cuMemGetAddressRange failed with CUresult %d", (int)r);
    cudaIpcMemHandle_t h;
    CUDA_TRY(cudaIpcGetMemHandle(&h, (void *)base));
    memcpy(handle64, &h, 64);
    *offset = (size_t)((CUdeviceptr)dev_ptr - base);
    return FCMA_OK;
}
extern "C" int fcma_ipc_open_handle(const void *handle64, void **base_ptr)
{
    if (!handle64 || !base_ptr) return fail(FCMA_EINVAL, "fcma_ipc_open_handle: null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CUDA_TRY(cudaIpcOpenMemHandle(base_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return FCMA_OK;
}
extern "C" int fcma_ipc_close_handle(void *base_ptr)
{
    if (!base_ptr) return FCMA_OK;
    CUDA_TRY(cudaIpcCloseMemHandle(base_ptr));
    return FCMA_OK;
}
extern "C" int fcma_peer_copy_async(void *dst, const void *src, size_t bytes, void *stream)
{
    if (!dst || !src) return fail(FCMA_EINVAL, "fcma_peer_copy_async: null pointer");
    CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return FCMA_OK;
}

extern "C" int fcma_host_within_subject_norm(float *corr_host, long n0, int E, long n2, int eps, int device)
{
    if (!corr_host || n0 <= 0 || E <= 0 || n2 <= 0) return fail(FCMA_EINVAL, "fcma_host_within_subject_norm: bad shape");
    if (fcma_device_count() == 0) return fail(FCMA_ENODEV, "no sm_90 device");
    DeviceGuard guard;
    CUDA_TRY(cudaSetDevice(device));
    DevBuf d;
    size_t bytes = (size_t)n0 * E * n2 * sizeof(float);
    CUDA_TRY(d.alloc(bytes));
    CUDA_TRY(cudaMemcpy(d.p, corr_host, bytes, cudaMemcpyHostToDevice));
    int rc = fcma_within_subject_norm((float *)d.p, n0, E, n2, eps, 0);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpy(corr_host, d.p, bytes, cudaMemcpyDeviceToHost));
    return FCMA_OK;
}
