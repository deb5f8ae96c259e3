// What one SM's TMA unit sustains for the tile shapes of the FFT passes (no FFT): persistent kernel, one CTA per SM, a ring of NS
// 64 KiB shared-memory stages; one thread queues tensor / bulk loads, another one stores.  Modes: load only, store only, load->store.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/tmabw tools/tmabw.cu  ; run on the GPU.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>

#define CK(x)                                                                                     \
    do {                                                                                          \
        cudaError_t e_ = (x);                                                                     \
        if (e_ != cudaSuccess) {                                                                  \
            std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            std::exit(1);                                                                         \
        }                                                                                         \
    } while (0)

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t ph) {
    asm volatile(
        "{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(s32(b)), "r"(ph)
        : "memory");
}
__device__ __forceinline__ void t_g2s(void* dst, const void* map, int x, int y, int z, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(s32(dst)),
                 "l"(map), "r"(s32(bar)), "r"(x), "r"(y), "r"(z)
                 : "memory");
}
__device__ __forceinline__ void t_s2g(const void* map, int x, int y, int z, const void* src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(s32(src)), "r"(x), "r"(y), "r"(z)
                 : "memory");
}
__device__ __forceinline__ void b_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(dst)), "l"(src), "r"(bytes),
                 "r"(s32(bar))
                 : "memory");
}
__device__ __forceinline__ void b_s2g(void* dst, const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(s32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

struct Params {
    CUtensorMap map_in, map_out;  // [slab][rows][cols] with box [1][box_rows][box_cols]
    const char* in;
    char* out;
    uint32_t tiles;          // tiles in the buffer (tile t: part t % split, then column block, then slab)
    uint32_t tiles_per_slab;
    uint32_t split;          // a column block of the slab is moved as `split` tiles of consecutive rows (adjacent CTAs)
    uint32_t total;          // tiles to move (wraps over `tiles`)
    uint32_t box_cols_elems; // inner box extent in ELEMENTS of the map's data type
    uint32_t box_rows, nbox; // tile = nbox boxes stacked along rows
    uint32_t mode;           // 0 tensor load only, 1 tensor store only, 2 tensor load -> tensor store, 3 bulk load only, 4 bulk store only,
                             // 5 bulk load -> bulk store, 6 tensor load -> bulk store, 7 bulk load -> tensor store
};
constexpr int NS = 3;
constexpr uint32_t TILE = 65536;

__global__ void __launch_bounds__(128, 1) k_tma(const __grid_constant__ Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char* base = smem + ((128u - (s32(smem) & 127u)) & 127u);
    uint64_t* full = reinterpret_cast<uint64_t*>(base + NS * TILE);
    uint64_t* empty = full + NS;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const bool do_load = p.mode == 0 || p.mode == 2 || p.mode == 3 || p.mode == 5 || p.mode == 6 || p.mode == 7;
    const bool do_store = p.mode == 1 || p.mode == 2 || p.mode == 4 || p.mode == 5 || p.mode == 6 || p.mode == 7;
    const bool bulk_load = p.mode == 3 || p.mode == 5 || p.mode == 7;
    const bool bulk_store = p.mode == 4 || p.mode == 5 || p.mode == 6;
    const uint32_t box_bytes = TILE / p.nbox;
    if (threadIdx.x == 0 && do_load) {  // loader
        uint32_t i = 0;
        for (uint32_t t = blockIdx.x; t < p.total; t += gridDim.x, ++i) {
            const uint32_t s = i % NS, ph = (i / NS) & 1u;
            mbar_wait(&empty[s], ph ^ 1u);
            const uint32_t tt = t % p.tiles, cb = tt / p.split, row0 = (tt % p.split) * p.nbox * p.box_rows;
            mbar_expect(&full[s], TILE);
            if (bulk_load)
                b_g2s(base + s * TILE, p.in + (size_t)tt * TILE, TILE, &full[s]);
            else
                for (uint32_t k = 0; k < p.nbox; ++k)
                    t_g2s(base + s * TILE + k * box_bytes, &p.map_in, (int)((cb % p.tiles_per_slab) * p.box_cols_elems), (int)(row0 + k * p.box_rows),
                          (int)(cb / p.tiles_per_slab), &full[s]);
        }
    }
    if (threadIdx.x == 32) {  // storer (or the consumer that just frees the stage)
        uint32_t i = 0;
        for (uint32_t t = blockIdx.x; t < p.total; t += gridDim.x, ++i) {
            const uint32_t s = i % NS, ph = (i / NS) & 1u;
            if (do_load) mbar_wait(&full[s], ph);
            if (do_store) {
                const uint32_t tt = t % p.tiles, cb = tt / p.split, row0 = (tt % p.split) * p.nbox * p.box_rows;
                if (bulk_store)
                    b_s2g(p.out + (size_t)tt * TILE, base + s * TILE, TILE);
                else
                    for (uint32_t k = 0; k < p.nbox; ++k)
                        t_s2g(&p.map_out, (int)((cb % p.tiles_per_slab) * p.box_cols_elems), (int)(row0 + k * p.box_rows), (int)(cb / p.tiles_per_slab),
                              base + s * TILE + k * box_bytes);
                commit();
                wait_read0();
            }
            if (do_load) mbar_arrive(&empty[s]);
        }
        wait_all0();
    }
}

typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                              const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
    encode_fn enc = (encode_fn)fp;
    const size_t BIG = 4ull << 30, SMALL = 32ull << 20;
    char *a, *b;
    CK(cudaMalloc(&a, BIG));
    CK(cudaMalloc(&b, BIG));
    CK(cudaMemset(a, 1, BIG));
    CK(cudaMemset(b, 1, BIG));
    CK(cudaFuncSetAttribute(k_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, NS * TILE + 1024));
    int sms = 0, khz = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
    const double ghz = khz / 1e6;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const char* mode_name[8] = {"tensor load", "tensor store", "tensor ld->st", "bulk load", "bulk store", "bulk ld->st", "tensor ld->bulk st", "bulk ld->tensor st"};
    // column blocks of a slab (`rows` rows of 8 KiB): rows x row bytes, moved as `split` 64 KiB tiles of rows / split rows each
    // (1024 x 128 B in two halves: the 16-column block of a 1024-row slab that two adjacent CTAs share)
    struct Shape { uint32_t rows, row_bytes, split; };
    const Shape shapes[] = {{1024, 64, 1}, {512, 128, 1}, {1024, 128, 2}, {256, 256, 1}, {128, 512, 1}};
    for (size_t buf : {SMALL, BIG}) {
        for (int esz : {4, 8}) {
            for (const Shape& sh : shapes) {
                Params p;
                const uint64_t slab_row_bytes = 8192;  // a slab = rows x 8 KiB matrix
                const uint64_t slab_bytes = (uint64_t)sh.rows * slab_row_bytes;
                const uint64_t slabs = buf / slab_bytes;
                p.tiles_per_slab = (uint32_t)(slab_row_bytes / sh.row_bytes);
                p.split = sh.split;
                p.tiles = (uint32_t)(slabs * p.tiles_per_slab * sh.split);
                p.total = (uint32_t)((4ull << 30) / TILE);
                p.box_cols_elems = sh.row_bytes / esz;
                const uint32_t tile_rows = sh.rows / sh.split;
                p.box_rows = tile_rows < 256 ? tile_rows : 256;
                p.nbox = tile_rows / p.box_rows;
                p.in = a;
                p.out = b;
                const cuuint64_t dims[3] = {slab_row_bytes / esz, sh.rows, slabs};
                const cuuint64_t strides[2] = {slab_row_bytes, slab_bytes};
                const cuuint32_t box[3] = {p.box_cols_elems, p.box_rows, 1};
                const cuuint32_t estr[3] = {1, 1, 1};
                const CUtensorMapDataType dt = esz == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT64;
                if (enc(&p.map_in, dt, 3, a, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS ||
                    enc(&p.map_out, dt, 3, b, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
                    std::printf("encode failed\n");
                    return 1;
                }
                for (uint32_t mode = 0; mode < 8; ++mode) {
                    if ((mode == 3 || mode == 4 || mode == 5) && !(esz == 4 && &sh == &shapes[0])) continue;  // bulk modes do not depend on the shape
                    p.mode = mode;
                    float best = 1e30f;
                    for (int r = 0; r < 3; ++r) {
                        CK(cudaEventRecord(e0));
                        k_tma<<<sms, 128, NS * TILE + 1024>>>(p);
                        CK(cudaEventRecord(e1));
                        CK(cudaEventSynchronize(e1));
                        float ms;
                        CK(cudaEventElapsedTime(&ms, e0, e1));
                        if (ms < best) best = ms;
                    }
                    CK(cudaGetLastError());
                    const double bytes = (double)p.total * TILE * ((mode == 2 || mode >= 5) ? 2 : 1);
                    std::printf("%s  elem %dB  tile %4u x %3uB /%u  %-18s %8.1f GB/s total = %6.1f GB/s per SM (%5.1f B/clk @%.2fGHz)\n", buf == SMALL ? "L2 " : "HBM", esz,
                                sh.rows, sh.row_bytes, sh.split, mode_name[mode], bytes / best / 1e6, bytes / best / 1e6 / sms, bytes / best / 1e6 / sms / ghz, ghz);
                }
            }
        }
    }
    return 0;
}
