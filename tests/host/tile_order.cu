// Host-side check (no GPU needed) of the GEMM tile order: gemm_tile_coords must be a bijection of [0, num_m * num_n) onto the
// tile grid for every group size, and a wave of 132 consecutive tiles (one per H100 SM) of the grouped order must span fewer m-tiles.
// Built and run by tests/test_host_logic.py with nvcc (host code only).
#include <cstdio>
#include <vector>
#include <cuda_bf16.h>
#include "../../mmada_parallel_b200/csrc/ptx.cuh"
#include "../../mmada_parallel_b200/csrc/gemm_epilogue.cuh"

int main() {
    int checked = 0;
    for (int num_m : {1, 2, 19, 37, 46, 57, 58, 76, 113}) {
        for (int num_n : {1, 16, 22, 48, 96, 526}) {
            for (int g : {0, 1, 2, 7, 19, 29, 40, num_m, num_m + 5}) {
                std::vector<int> seen(num_m * num_n, 0);
                for (int tl = 0; tl < num_m * num_n; ++tl) {
                    int m = -1, n = -1;
                    mmdp::gemm_tile_coords(tl, num_m, num_n, g, m, n);
                    if (m < 0 || m >= num_m || n < 0 || n >= num_n) { printf("FAIL range num_m=%d num_n=%d g=%d tl=%d -> (%d,%d)\n", num_m, num_n, g, tl, m, n); return 1; }
                    if (seen[m * num_n + n]++) { printf("FAIL duplicate num_m=%d num_n=%d g=%d tl=%d -> (%d,%d)\n", num_m, num_n, g, tl, m, n); return 1; }
                }
                ++checked;
            }
        }
    }
    // wave shape at the bench-adjacent shape: 57 m-tiles x 48 n-tiles, first wave of 132 tiles
    auto span = [](int g) {
        int mmin = 1 << 30, mmax = -1;
        for (int tl = 0; tl < 132; ++tl) { int m, n; mmdp::gemm_tile_coords(tl, 57, 48, g, m, n); mmin = m < mmin ? m : mmin; mmax = m > mmax ? m : mmax; }
        return mmax - mmin + 1;
    };
    if (span(0) != 57 || span(29) != 29) { printf("FAIL wave span %d %d\n", span(0), span(29)); return 1; }
    printf("OK %d configurations\n", checked);
    return 0;
}
