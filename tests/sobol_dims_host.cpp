// Host build of the direction numbers of particles_b200/csrc/smcb_sqmc.cuh: the committed table of the first
// kSobolTabDim dimensions and the expansion of any dimension from Joe and Kuo's initial numbers, so that
// tests/test_ffbs_qmc_host.py can compare the two.
//   g++ -O2 -shared -fPIC -I particles_b200/csrc tests/sobol_dims_host.cpp
#include <cmath>
#include <cstdint>

#define SMCB_SQMC_HOST_TEST 1
#define __device__
#define __host__
#define __forceinline__ inline
using std::fabs; using std::floor; using std::fma; using std::sqrt;

#include "smcb_sqmc.cuh"

using namespace smcb::sqmc;

extern "C" {

int sd_max_dim() { return kSobolMaxDim; }
int sd_tab_dim() { return kSobolTabDim; }

// the 30 direction numbers of dimension j: from the table (tab != 0, j < kSobolTabDim) or expanded (1 <= j)
void sd_dirs(int j, int tab, uint32_t *out) {
    if (tab) {
        for (int k = 0; k < kSobolBits; k++) out[k] = kSobolDirs[j][k];
    } else {
        sobol_expand(j, out);
    }
}

}  // extern "C"
