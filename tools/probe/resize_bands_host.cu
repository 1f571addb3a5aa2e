// Host-side check of the band construction in pix2pix3d_b200/csrc/resize.cu: prints the dense forward matrix built from the
// forward bands and the dense matrix built from the transposed bands (which must be its transpose).
//   nvcc -std=c++17 -o resize_bands_host tools/probe/resize_bands_host.cu && ./resize_bands_host 128 512 1
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../pix2pix3d_b200/csrc/resize.cu"

namespace p3d { int sm_count() { return 1; } }

int main(int argc, char** argv) {
    const int in = atoi(argv[1]), out = atoi(argv[2]), aa = atoi(argv[3]);
    for (int transposed = 0; transposed < 2; ++transposed) {
        p3d::ResizeAxis a = p3d::make_axis(in, out, aa, transposed);
        std::vector<float> w(a.K);
        const int rows = transposed ? in : out;
        printf("%d %d\n", rows, a.K);
        for (int r = 0; r < rows; ++r) {
            int s = 0, c = 0;
            p3d::make_band(a, transposed, r, s, c, w.data());
            printf("%d %d", s, c);
            for (int k = 0; k < c; ++k) printf(" %.9g", w[k]);
            printf("\n");
        }
    }
    return 0;
}
