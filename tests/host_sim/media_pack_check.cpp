// Host build of the scene pack (toypathtracer_b200/csrc/tpt_scene_pack.h), exactly as tpt_set_scene and tpt_set_media run
// it, for tests/test_media_api.py: g++ -shared, called through ctypes.
#include "../../toypathtracer_b200/csrc/tpt_scene_pack.h"
#include <string.h>

// The media section is found from offMatRi and the count: the layout the trace kernels take does not grow.
static_assert(sizeof(tpt::SceneBlobLayout) == 116, "SceneBlobLayout size");

extern "C" {

// Packs count spheres (20 B) and materials (36 B) with emissives (null: derived) and nMedia media records (null: none)
// under sceneFlags. Copies the blob into out (at most cap bytes) and the layout into layout116; returns the blob's size.
long long pack_blob(const void* spheres, const void* mats, int count, const int* emissives, int nEmissives,
                    unsigned sceneFlags, const float* media5, int nMedia, unsigned char* out, long long cap, void* layout116)
{
    std::vector<unsigned char> blob;
    tpt::SceneBlobLayout L;
    int nLights = 0;
    tpt::pack_scene_blob((const tpt::Sphere20*)spheres, (const tpt::Material36*)mats, count, emissives, nEmissives, blob, L,
                         nLights, sceneFlags, media5, nMedia);
    memcpy(out, blob.data(), blob.size() < (size_t)cap ? blob.size() : (size_t)cap);
    memcpy(layout116, &L, sizeof(L));
    return (long long)blob.size();
}

long long media_offset_of(unsigned offMatRi, int count) { return (long long)tpt::media_offset(offMatRi, count); }
long long media_bytes_of(int count) { return (long long)tpt::media_bytes(count); }

}
