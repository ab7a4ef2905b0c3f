// Host build of the emission-layer table builder (toypathtracer_b200/csrc/tpt_env_tables.h), exactly as
// tpt_set_emission_textures runs it, for tests/test_emission_texture_sampling_api.py: g++ -shared, called through ctypes.
#include "../../toypathtracer_b200/csrc/tpt_env_tables.h"
#include "../../toypathtracer_b200/csrc/tpt_types.h"

// The kernels find the layers' tables through TexSet's spare word: neither the set nor the layout the trace kernels take
// grows.
static_assert(sizeof(tpt::TexSet) == 32, "TexSet size");
static_assert(sizeof(tpt::SceneBlobLayout) == 116, "SceneBlobLayout size");

extern "C" {

// texels: L * W * H float4 (R, G, B read; alpha receives each cell's realised probability, 0 in a layer without
// tables). tables: L blocks of H + W * H {prob, alias} pairs. Returns 1 when some layer is sampleable.
int emit_tables_check(float* texels, int W, int H, int L, void* tables)
{
    return emit_build_tables(texels, W, H, L, static_cast<EnvAlias*>(tables)) ? 1 : 0;
}

// The slot size tpt_set_emission_textures allocates, and where the tables start in it.
long long emit_slot_size(int W, int H, int L, int S) { return (long long)emit_slot_bytes(W, H, L, S); }
long long emit_tables_at(int W, int H, int L, int S) { return (long long)emit_table_offset(W, H, L, S); }
int emit_no_tables() { return kEmitNoTables; }
long long scene_layout_size() { return (long long)sizeof(tpt::SceneBlobLayout); }

}
