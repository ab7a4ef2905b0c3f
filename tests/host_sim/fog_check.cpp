// Host build of the fog's pack, chord and phase function (toypathtracer_b200/csrc/tpt_scene_pack.h, tpt_fog.h), exactly as
// tpt_set_fog and the fast kernels run them, for tests/test_fog_api.py: g++ -shared, called through ctypes.
#include "../../toypathtracer_b200/csrc/tpt_scene_pack.h"
#include <string.h>

// The fog section is found from offMatRi, the count and the flags: the layout the trace kernels take does not grow.
static_assert(sizeof(tpt::SceneBlobLayout) == 116, "SceneBlobLayout size");

extern "C" {

// Packs count spheres (20 B) and materials (36 B) with emissives (null: derived), nMedia media records (null: none) and
// the fog record fog9 (null: none) under sceneFlags. Copies the blob into out (at most cap bytes) and the layout into
// layout116; returns the blob's size.
long long pack_blob_fog(const void* spheres, const void* mats, int count, const int* emissives, int nEmissives,
                        unsigned sceneFlags, const float* media5, int nMedia, const float* fog9, unsigned char* out,
                        long long cap, void* layout116)
{
    std::vector<unsigned char> blob;
    tpt::SceneBlobLayout L;
    int nLights = 0;
    tpt::pack_scene_blob((const tpt::Sphere20*)spheres, (const tpt::Material36*)mats, count, emissives, nEmissives, blob, L,
                         nLights, sceneFlags, media5, nMedia, fog9);
    memcpy(out, blob.data(), blob.size() < (size_t)cap ? blob.size() : (size_t)cap);
    memcpy(layout116, &L, sizeof(L));
    return (long long)blob.size();
}

long long fog_offset_of(unsigned offMatRi, int count, unsigned flags) { return (long long)tpt::fog_offset(offMatRi, count, flags); }

// fog_chord for n segments seg[10 i ..] = {o.xyz, d.xyz, t, c.xyz} with radius R[i]: lengths into L, starts into tin.
void fog_chords(const float* seg, const float* R, int n, float* L, float* tin)
{
    for (int i = 0; i < n; ++i)
    {
        const float* s = seg + 10 * i;
        L[i] = tpt::fog_chord(s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7], s[8], s[9], R[i], tin + i);
    }
}

// hg_phase at n cosines.
void hg_phases(const float* cosT, int n, float g, float* out)
{
    for (int i = 0; i < n; ++i) out[i] = tpt::hg_phase(cosT[i], g);
}

}
