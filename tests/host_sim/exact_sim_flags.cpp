// Test-only: exact_sim.cpp (the HOST build of tpt_integrator.cuh) with the scene's kScene* bits settable, the way
// tpt_set_option's scene switches reach tpt_set_scene: sim_set_scene_flags(bits) applies to the following sim_render_*
// calls (default 0). exact_sim.cpp packs its scenes with pack_scene_blob()'s default flags; the macro below appends the
// flags argument to those calls and leaves the rest of that file as it is. Never linked into the product library.
// Build: g++ -O2 -std=c++17 -ffp-contract=off -mfma, like exact_sim.cpp.
#include "../../toypathtracer_b200/csrc/tpt_scene_pack.h"

static unsigned g_sceneFlags = 0;
extern "C" void sim_set_scene_flags(unsigned flags) { g_sceneFlags = flags; }

#define pack_scene_blob(...) pack_scene_blob(__VA_ARGS__, g_sceneFlags)
#include "exact_sim.cpp"
#undef pack_scene_blob
