// Host build of the occupancy distance transform of pvb_device.cuh (pvb_occupancy_sdf, OccupancySDF) behind a small C
// interface for tests/test_occupancy_sdf_cpu.py.
//   simedt_occupancy_sdf runs the three passes and the record writer of pvb_occupancy_sdf over host memory: the bit
//   words edt_z_kernel builds with ballots, edt_line_nearest for every position of every z line, edt_envelope for
//   every y line and then every x line (the stack in a host buffer, stride 1), edt_record per voxel.  Both states are
//   carried as in the kernels: state 0 takes the occupied voxels as sites, state 1 the free ones.
// Test infrastructure only.
#include <vector>

#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

// occ uint8 [nx][ny][nz]; outputs as pvb_occupancy_sdf (each may be null)
extern "C" void simedt_occupancy_sdf(const unsigned char *occ, const int *dims, float resolution, int *out_sqdist,
                                     int *out_site, float *out_table) {
    const int nx = dims[0], ny = dims[1], nz = dims[2];
    const long long n_vox = (long long)nx * ny * nz;
    std::vector<EdtPair> a(2 * n_vox), b(2 * n_vox);
    const int n_words = (nz + 31) >> 5;
    for (long long line = 0; line < (long long)nx * ny; ++line) {
        const long long base = line * nz;
        uint32_t words[2][kEdtMaxDim / 32] = {};
        for (int p = 0; p < nz; ++p) words[occ[base + p] != 0 ? 0 : 1][p >> 5] |= 1u << (p & 31);
        for (int p = 0; p < nz; ++p)
            for (int t = 0; t < 2; ++t) {
                const int r = edt_line_nearest(words[t], n_words, p);
                a[t * n_vox + base + p] = r < 0 ? EdtPair{-1, -1} : EdtPair{(p - r) * (p - r), (int)(base + r)};
            }
    }
    std::vector<EdtPair> stk(kEdtMaxDim);
    auto pass = [&](const std::vector<EdtPair> &in, std::vector<EdtPair> &out, int n, long long stride) {
        const long long n_lines = n_vox / n;
        for (int t = 0; t < 2; ++t)
            for (long long l = 0; l < n_lines; ++l) {
                const long long base = (l / stride) * (stride * n) + l % stride;
                edt_envelope(in.data() + t * n_vox + base, out.data() + t * n_vox + base, stride, n, stk.data(), 1);
            }
    };
    pass(a, b, ny, nz);
    pass(b, a, nx, (long long)ny * nz);
    for (long long c = 0; c < n_vox; ++c) {
        const bool o = occ[c] != 0;
        const EdtPair e = a[(o ? n_vox : 0) + c];
        if (out_sqdist) out_sqdist[c] = e.d;
        if (out_site) out_site[c] = e.s;
        if (out_table) {
            const int ci = (int)c, s = e.s < 0 ? 0 : e.s;
            const float4 r = edt_record(e.d, o, ci / nz / ny, (ci / nz) % ny, ci % nz, s / nz / ny, (s / nz) % ny,
                                        s % nz, resolution);
            out_table[4 * c] = r.x; out_table[4 * c + 1] = r.y; out_table[4 * c + 2] = r.z; out_table[4 * c + 3] = r.w;
        }
    }
}
