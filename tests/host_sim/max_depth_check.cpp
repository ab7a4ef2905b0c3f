// Host build of the "max_depth" encoding (toypathtracer_b200/csrc/tpt_types.h), exactly as begin_call writes it into a
// call's flags and the kernels' scene views read it back, for tests/test_max_depth_api.py: g++ -shared, called through
// ctypes.
#include "../../toypathtracer_b200/csrc/tpt_scene_pack.h"

// The value travels in the call's copy of the flags: the layout the trace kernels take does not grow.
static_assert(sizeof(tpt::SceneBlobLayout) == 116, "SceneBlobLayout size");

extern "C" {

unsigned depth_flags_of(int n) { return tpt::depth_flags(n); }
int max_depth_of(unsigned flags) { return tpt::scene_max_depth(flags); }
unsigned scene_depth_flag() { return tpt::kSceneDepth; }
unsigned ref_form_mask() { return tpt::kSceneRefForm; }
int ref_max_depth() { return tpt::kRefMaxDepth; }
int max_path_depth() { return tpt::kMaxPathDepth; }

// The max_depth a host scene view made from a layout with these flags carries (scene_view_from_blob).
int view_max_depth(unsigned flags)
{
    tpt::SceneBlobLayout L{};
    L.flags = flags;
    return tpt::scene_view_from_blob(nullptr, L, 1, 0).maxDepth;
}

}
