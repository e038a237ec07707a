// ht2_inflate.cu -- the device backend of ht2_inflate.h and ht2gpu_gunzip.
//
// Kernel organisation (DESIGN.md 5.2):
//   find     one CTA of 256 threads per chunk, one candidate bit offset per thread, rounds of 256 offsets until the
//            first start is found (the smallest offset of the round wins);
//   decode   one thread per chunk; its literal/length and distance tables (3.2 KB) in shared memory; as many threads
//            per CTA as keeps every SM busy;
//   window   one CTA, sequential over the chunks in order, parallel over the 32 KiB of each window;
//   replace  a grid over every symbol of every chunk;
//   crc      one thread per 4 KiB piece of a member's output in a chunk, a CRC table in shared memory; the pieces are
//            combined on the host (crc32_combine arithmetic on the piece values, no pass over the bytes).
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>

#include "ht2_inflate.h"

namespace {

__global__ void __launch_bounds__(256) ht2z_find_kernel(const uint8_t* src, uint64_t base, uint64_t end, uint64_t wb, uint64_t C,
                                                         uint64_t we, uint64_t* keys, uint32_t* kinds)
{
    __shared__ unsigned long long best;
    const uint32_t k = blockIdx.x + 1;
    const uint64_t r0 = (wb + k * C) * 8, r1 = (wb + (k + 1) * C < we ? wb + (k + 1) * C : we) * 8;
    if (threadIdx.x == 0) best = ~0ull;
    __syncthreads();
    for (uint64_t b0 = r0; b0 < r1; b0 += blockDim.x) {
        const uint64_t bit = b0 + threadIdx.x;
        if (bit < r1) {
            const uint32_t kind = ht2z_candidate(src, base, end, bit);
            if (kind) atomicMin(&best, (unsigned long long)(bit << 2 | kind));
        }
        __syncthreads();
        if (best != ~0ull) break;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        keys[k] = best == ~0ull ? HT2Z_NONE : (uint64_t)(best >> 2);
        kinds[k] = best == ~0ull ? (uint32_t)HT2Z_K_NONE : (uint32_t)(best & 3);
    }
}

__global__ void ht2z_decode_kernel(Ht2zChunk* ch, const int* ids, int nids, const uint8_t* src, uint64_t base, uint64_t end,
                                   bool final, uint16_t* sym, uint32_t slice)
{
    extern __shared__ Ht2zTables tabs[];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nids) return;
    const int id = ids[t];
    ht2z_run(ch[id], src, base, end, final, sym + (size_t)id * slice, tabs[threadIdx.x]);
}

__global__ void __launch_bounds__(1024) ht2z_window_kernel(const Ht2zChunk* ch, const int* ids, int m, const uint32_t* vld,
                                                            const uint16_t* sym, uint32_t slice, uint8_t* win, uint32_t* bad)
{
    uint32_t b = 0;
    for (int i = 0; i < m; i++) {
        const uint16_t* s = sym + (size_t)ids[i] * slice;
        const uint32_t n = ch[ids[i]].nout;
        const uint8_t* w = win + (size_t)i * HT2Z_WSIZE;
        uint8_t* o = win + (size_t)(i + 1) * HT2Z_WSIZE;
        for (uint32_t j = threadIdx.x; j < HT2Z_WSIZE; j += blockDim.x) o[j] = ht2z_next_win(j, s, n, w, vld[i], &b);
        __syncthreads();
    }
    if (b) atomicOr(bad, 1u);
}

__global__ void ht2z_replace_kernel(const Ht2zChunk* ch, const int* ids, const uint64_t* off, const uint32_t* vld, const uint16_t* sym,
                                    uint32_t slice, const uint8_t* win, uint8_t* out, uint32_t* bad)
{
    const int i = blockIdx.y;
    const uint32_t n = ch[ids[i]].nout;
    const uint16_t* s = sym + (size_t)ids[i] * slice;
    const uint8_t* w = win + (size_t)i * HT2Z_WSIZE;
    uint8_t* o = out + off[i];
    uint32_t b = 0;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) o[j] = ht2z_sym(s[j], w, vld[i], &b);
    if (b) atomicOr(bad, 1u);
}

__global__ void __launch_bounds__(256) ht2z_crc_kernel(const Ht2zPiece* pcs, int n, const uint8_t* out, uint32_t* crc)
{
    __shared__ uint32_t tab[256];
    tab[threadIdx.x] = ht2z_crc_byte(threadIdx.x);
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) crc[i] = ht2z_crc(0, out + pcs[i].off, pcs[i].len, tab);
}

#define ZK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) throw std::runtime_error(std::string(#call) + ": " + cudaGetErrorString(e_)); } while (0)

struct DeviceBackend {
    ht2gpu_gunzip_stats_t& S;
    cudaStream_t stream = NULL;
    cudaEvent_t e0 = NULL, e1 = NULL;
    uint8_t *dSrc = NULL, *dWin = NULL, *dOut = NULL;
    uint16_t* dSym = NULL;
    Ht2zChunk* dCh = NULL;
    uint64_t *dKeys = NULL, *dOff = NULL;
    uint32_t *dKinds = NULL, *dVld = NULL, *dPcrc = NULL, *dBad = NULL;
    Ht2zPiece* dPcs = NULL;
    int* dIds = NULL;
    uint64_t base = 0, end = 0;
    int nSM = 0;
    explicit DeviceBackend(ht2gpu_gunzip_stats_t& s) : S(s) {}
    template <class T> void alloc(T*& p, size_t n)
    {
        ZK(cudaMalloc((void**)&p, n * sizeof(T)));
        S.peak_device_bytes += n * sizeof(T);
    }
    void init(int device)
    {
        const Ht2zGeom& G = HT2Z_GEOM;
        ZK(cudaDeviceGetAttribute(&nSM, cudaDevAttrMultiProcessorCount, device));
        ZK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        ZK(cudaEventCreate(&e0)); ZK(cudaEventCreate(&e1));
        alloc(dSrc, G.maxWindowIn + G.lookahead);
        alloc(dSym, G.symBudget);
        alloc(dOut, G.symBudget);
        alloc(dWin, (size_t)(G.maxChunks + 1) * HT2Z_WSIZE);
        alloc(dCh, G.maxChunks);
        alloc(dKeys, G.maxChunks); alloc(dKinds, G.maxChunks);
        alloc(dOff, G.maxChunks + 1); alloc(dVld, G.maxChunks + 1);
        const size_t maxPieces = G.symBudget / HT2Z_PIECE + (size_t)G.maxChunks * (HT2Z_EV + 1);
        alloc(dPcs, maxPieces); alloc(dPcrc, maxPieces);
        alloc(dIds, G.maxChunks); alloc(dBad, 1);
        ZK(cudaMemsetAsync(dWin, 0, HT2Z_WSIZE, stream));
        ZK(cudaFuncSetAttribute(ht2z_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * (int)sizeof(Ht2zTables)));
    }
    ~DeviceBackend()
    {
        if (stream) cudaStreamSynchronize(stream);
        cudaFree(dSrc); cudaFree(dSym); cudaFree(dOut); cudaFree(dWin); cudaFree(dCh); cudaFree(dKeys); cudaFree(dKinds);
        cudaFree(dOff); cudaFree(dVld); cudaFree(dPcs); cudaFree(dPcrc); cudaFree(dIds); cudaFree(dBad);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
        if (stream) cudaStreamDestroy(stream);
    }
    template <class F> void timed(float& acc, F f)
    {
        ZK(cudaEventRecord(e0, stream));
        f();
        ZK(cudaGetLastError());
        ZK(cudaEventRecord(e1, stream));
        ZK(cudaEventSynchronize(e1));
        float ms = 0;
        ZK(cudaEventElapsedTime(&ms, e0, e1));
        acc += ms;
    }
    void setSrc(const uint8_t* p, uint64_t b, uint64_t e)
    {
        base = b; end = e;
        timed(S.ms_copy, [&] { ZK(cudaMemcpyAsync(dSrc, p, e - b, cudaMemcpyHostToDevice, stream)); });
    }
    void find(uint64_t wb, uint64_t C, uint32_t nc, uint64_t we, uint64_t* keys, uint32_t* kinds)
    {
        if (nc < 2) return;
        timed(S.ms_find, [&] {
            ht2z_find_kernel<<<nc - 1, 256, 0, stream>>>(dSrc, base, end, wb, C, we, dKeys, dKinds);
            ZK(cudaMemcpyAsync(keys + 1, dKeys + 1, (nc - 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
            ZK(cudaMemcpyAsync(kinds + 1, dKinds + 1, (nc - 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        });
    }
    void decode(Ht2zChunk* ch, uint32_t nc, const std::vector<int>& ids, uint32_t slice, bool final)
    {
        const int n = (int)ids.size();
        int tpb = 1;   // spread the chunks over every SM before putting several in one CTA
        while (tpb < 32 && n / (tpb * 2) >= 2 * nSM) tpb *= 2;
        timed(S.ms_decode, [&] {
            ZK(cudaMemcpyAsync(dCh, ch, nc * sizeof(Ht2zChunk), cudaMemcpyHostToDevice, stream));
            ZK(cudaMemcpyAsync(dIds, ids.data(), n * sizeof(int), cudaMemcpyHostToDevice, stream));
            ht2z_decode_kernel<<<(n + tpb - 1) / tpb, tpb, tpb * sizeof(Ht2zTables), stream>>>(dCh, dIds, n, dSrc, base, end, final, dSym, slice);
            ZK(cudaMemcpyAsync(ch, dCh, nc * sizeof(Ht2zChunk), cudaMemcpyDeviceToHost, stream));
        });
    }
    int resolve(const Ht2zChunk* ch, const std::vector<int>& L, const std::vector<uint64_t>& off, const std::vector<uint32_t>& vld,
                uint32_t slice, char* out, const std::vector<Ht2zPiece>& pcs, uint32_t* pcrc)
    {
        const int m = (int)L.size();
        uint32_t maxN = 0;
        for (int i = 0; i < m; i++) maxN = ch[L[i]].nout > maxN ? ch[L[i]].nout : maxN;
        uint32_t bad = 0;
        timed(S.ms_window, [&] {
            ZK(cudaMemcpyAsync(dIds, L.data(), m * sizeof(int), cudaMemcpyHostToDevice, stream));
            ZK(cudaMemcpyAsync(dOff, off.data(), (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, stream));
            ZK(cudaMemcpyAsync(dVld, vld.data(), (m + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
            ZK(cudaMemsetAsync(dBad, 0, sizeof(uint32_t), stream));
            ht2z_window_kernel<<<1, 1024, 0, stream>>>(dCh, dIds, m, dVld, dSym, slice, dWin, dBad);
        });
        if (maxN) timed(S.ms_replace, [&] {
            const uint32_t gx = (maxN + 255) / 256 < 64 ? (maxN + 255) / 256 : 64;
            ht2z_replace_kernel<<<dim3(gx, m), 256, 0, stream>>>(dCh, dIds, dOff, dVld, dSym, slice, dWin, dOut, dBad);
        });
        const int np = (int)pcs.size();
        if (np) timed(S.ms_crc, [&] {
            ZK(cudaMemcpyAsync(dPcs, pcs.data(), np * sizeof(Ht2zPiece), cudaMemcpyHostToDevice, stream));
            ht2z_crc_kernel<<<(np + 255) / 256, 256, 0, stream>>>(dPcs, np, dOut, dPcrc);
        });
        timed(S.ms_copy, [&] {
            ZK(cudaMemcpyAsync(out, dOut, off[m], cudaMemcpyDeviceToHost, stream));
            if (np) ZK(cudaMemcpyAsync(pcrc, dPcrc, np * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
            ZK(cudaMemcpyAsync(&bad, dBad, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
        });
        return (int)bad;
    }
    void carry(uint32_t m)   // the window after the last kept chunk is the first window of the next round
    {
        ZK(cudaMemcpyAsync(dWin, dWin + (size_t)m * HT2Z_WSIZE, HT2Z_WSIZE, cudaMemcpyDeviceToDevice, stream));
    }
};

thread_local std::string tErr;
}   // namespace

extern "C" const char* ht2gpu_gunzip_error(void) { return tErr.c_str(); }

// The device inflate into any Ht2zOut (the read pipeline streams into its source buffer); error text in err.
int ht2_gunzip_to(int device, const void* src, size_t n, uint32_t chunkBytes, Ht2zOut& out, size_t* outLen,
                  ht2gpu_gunzip_stats_t* stats, std::string& err)
{
    ht2gpu_gunzip_stats_t S;
    memset(&S, 0, sizeof(S));
    if (stats) *stats = S;
    *outLen = 0;
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(device) != cudaSuccess) {
        cudaGetLastError();
        err = "ht2gpu_gunzip: no usable CUDA device " + std::to_string(device);
        return HT2GPU_ERR_CUDA;
    }
    int rc;
    try {
        DeviceBackend be(S);
        be.init(device);
        rc = ht2z_gunzip_to(be, (const uint8_t*)src, n, chunkBytes, out, outLen, S, err);
    } catch (const std::exception& e) {
        *outLen = 0;
        err = std::string("ht2gpu_gunzip: ") + e.what();
        rc = HT2GPU_ERR_CUDA;
    }
    cudaSetDevice(prev);
    if (stats) *stats = S;
    return rc;
}

extern "C" int ht2gpu_gunzip(int device, const void* src, size_t n, const ht2gpu_gunzip_opts_t* opts, char** out, size_t* out_len,
                             ht2gpu_gunzip_stats_t* stats)
{
    tErr.clear();
    if (stats) memset(stats, 0, sizeof(*stats));
    if ((!src && n) || !out || !out_len) { tErr = "ht2gpu_gunzip: invalid arguments"; return HT2GPU_ERR_ARG; }
    *out = NULL; *out_len = 0;
    Ht2zMallocOut O((const uint8_t*)src, n);
    const int rc = ht2_gunzip_to(device, src, n, opts ? opts->chunk_bytes : 0, O, out_len, stats, tErr);
    if (rc == HT2GPU_OK) *out = O.release();
    else *out_len = 0;
    return rc;
}
