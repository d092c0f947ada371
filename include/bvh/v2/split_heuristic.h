// <bvh/v2/split_heuristic.h> — same include path as the reference header of that name; the declarations live in
// <bvh/v2/b200_surface.h> (the reference's C++ surface re-authored on top of the CUDA engine).
#pragma once
#include <bvh/v2/b200_surface.h>
