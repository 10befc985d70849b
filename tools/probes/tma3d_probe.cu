// Development probe: cp.async.bulk.tensor 2-D / 3-D loads with the geometry of the final inverse level.
// nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -I../../cineform-sdk_b200/csrc tma3d_probe.cu ../../cineform-sdk_b200/csrc/cfb_tma.cu -o tma3d_probe
#include <cstdio>
#include <vector>
#include "cfb_tma.cuh"
using namespace cfb;

struct alignas(64) Maps { CUtensorMap m[4]; };
struct alignas(64) BigMaps { CUtensorMap m[100]; };

template <class M>
__global__ void k(const __grid_constant__ M tm, int idx2, int idx3, int mode, int x, int y, unsigned *out)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const unsigned base = smem_u32(smem), bar = base + 8192;
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
        unsigned tx = 0;
        if (mode & 1) tx += 512;
        if (mode & 2) tx += 1536;
        mbar_expect_tx(bar, tx);
        if (mode & 1) tma_load_2d(base, &tm.m[idx2], x, y, bar);
        if (mode & 2) tma_load_3d(base + 512, &tm.m[idx3], x, y, 0, bar);
    }
    __syncwarp();
    mbar_wait(bar, 0);
    for (int i = threadIdx.x; i < 512; i += 32) out[i] = lds32(base + 4 * i);
}

int main()
{
    const int W = 960, H = 540, pitch = 1920;
    const size_t band = (size_t)pitch * H;
    std::vector<unsigned short> h(4 * band / 2);
    for (size_t i = 0; i < h.size(); i++) h[i] = (unsigned short)((i / (band / 2)) * 10000 + ((i % (band / 2)) / (pitch / 2)) * 8 + (i % (pitch / 2)) % 8);
    unsigned char *d; cudaMalloc(&d, 4 * band); cudaMemcpy(d, h.data(), 4 * band, cudaMemcpyHostToDevice);
    unsigned *o; cudaMalloc(&o, 2048);
    Maps tm; BigMaps big;
    printf("enc2d %d\n", (int)tmap_encode_2d(&tm.m[0], d, W * 2, H, pitch, 256, 2));
    printf("enc3d %d\n", (int)tmap_encode_3d(&tm.m[1], d + band, W * 2, H, pitch, 3, band, 256, 2, 3));
    big.m[90] = tm.m[0]; big.m[91] = tm.m[1];
    for (int xs = 0; xs < 2; xs++)
    for (int big_params = 0; big_params < 2; big_params++)
    for (int mode = 1; mode <= 3; mode++) {
        const int x = xs ? -2 : -4;
        cudaMemset(o, 0, 2048);
        if (big_params) k<BigMaps><<<1, 32, 8256>>>(big, 90, 91, mode, x, 5, o);
        else k<Maps><<<1, 32, 8256>>>(tm, 0, 1, mode, x, 5, o);
        cudaError_t e = cudaDeviceSynchronize();
        unsigned r[512]; cudaMemcpy(r, o, 2048, cudaMemcpyDeviceToHost);
        printf("x %d big %d mode %d: %s | 2d row0: %08x %08x %08x row1: %08x | 3d b0r0: %08x %08x %08x b1r0 %08x b2r1 %08x\n", x, big_params, mode, cudaGetErrorString(e),
               r[0], r[1], r[2], r[64], r[128], r[129], r[130], r[128 + 128], r[128 + 256 + 64]);
        if (e != cudaSuccess) return 1;
    }
    return 0;
}
