/* rama_blur.cpp — TEST INFRASTRUCTURE: the reference's own Ramachandran blur, compiled unmodified.
 *
 * VIAMD's density task (src/components/ramachandran/ramachandran.cpp:1277-1370) blurs its 512 x 512 RGBA32F map with blur_density_gaussian
 * (:368-387: boxes_for_gauss + three box passes along the rows, a transpose, three along the columns, a transpose). That code is C++ inside the
 * application, so oracle/rama.mk cuts the block from `blur_rows_acc` to `blur_density_gaussian` out of the reference source at build time into
 * _ref/rama_blur.inc (never committed) and it is included here as it is; rama_harness.c calls it through the two C entry points below. */
#include <core/md_common.h>
#include <core/md_allocator.h>
#include <core/md_vec_math.h>

#include "rama_blur.inc"

extern "C" void ref_rama_boxes_for_gauss(int box_w[3], float sigma) { boxes_for_gauss(box_w, 3, sigma); }
extern "C" void ref_rama_blur_density_gaussian(float* rgba, int dim, float sigma) { blur_density_gaussian((vec4_t*)rgba, dim, sigma); }
