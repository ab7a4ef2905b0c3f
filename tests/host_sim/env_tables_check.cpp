// Host build of the environment-sampling table builder (toypathtracer_b200/csrc/tpt_env_tables.h), exactly as
// tpt_set_environment runs it, for tests/test_environment_sampling_api.py: g++ -shared, called through ctypes.
#include "../../toypathtracer_b200/csrc/tpt_env_tables.h"
#include <cstring>

extern "C" {

// texels: W * H float4 (R, G, B read; alpha receives each cell's realised probability when the map is sampleable).
// rows: H {prob, alias} pairs, cols: W * H, weights: W * H doubles (the pinned weight). Returns 1 when sampleable.
int env_tables_check(float* texels, int W, int H, void* rows, void* cols, double* weights)
{
    std::vector<double> w;
    env_weights(texels, W, H, w);
    std::memcpy(weights, w.data(), w.size() * sizeof(double));
    return env_build_tables(texels, W, H, static_cast<EnvAlias*>(rows), static_cast<EnvAlias*>(cols)) ? 1 : 0;
}

// The slot size tpt_set_environment allocates.
long long env_slot_size(int W, int H) { return (long long)env_slot_bytes(W, H); }

}
