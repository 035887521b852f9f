// Test hooks of the score + top-k row store (score.cu) that the diagnostic entry points (debug.cu) reach.
#pragma once
#include "common.cuh"

namespace mb {
namespace score {

// force_streamed: 1 makes every later scan of `ix` run the streamed-query kernel whatever its dim, 0 restores the
// library's rule (streamed only above 1024), -1 leaves the setting as it is.  *last_kernel (when not NULL) receives
// the kernel the last scan ran: 0 resident query block, 1 streamed, -1 no scan yet.
void debug_scan_kernel(b200_index* ix, int force_streamed, int* last_kernel);

// What the last scan of `ix` left on the device, for its query group (see b200_debug_index_last_scan).
void debug_last_scan(b200_index* ix, int* nq, int* grid, float* eps, float* queries, float* list_score,
                     int32_t* list_row, int32_t* list_doc);

}  // namespace score
}  // namespace mb
