// TEST INFRASTRUCTURE: host emulation of the character boxes in page pixels (DESIGN 4.20).  Compiles the bodies shared
// with the CUDA kernel (advancedliteratemachinery_b200/csrc/rec_box_core.h) as plain C++ and runs rec_box_kernel's
// work word by word: decode_seq's walk over the steps in order (the kernel numbers the same kept steps by ballots), the
// same char_box body for each kept step, zeros past the character count.  Built on the fly by
// tests/test_page_char_boxes_cpu.py (g++ -O1 -ffp-contract=off); never part of libalm_ocr.so.
#include <stdint.h>

#include <vector>

#include "../../advancedliteratemachinery_b200/csrc/rec_box_core.h"

using namespace alm;

extern "C" {

// alm_omni_char_boxes on the host (arguments validated by the caller)
void emu_char_boxes(long N, int L, const double* polys, const int64_t* rec, const float* loc, const int* frame_index,
                    int F, const int* frames, int64_t pad, int64_t eos, int* n_chars, int* step, double* centre,
                    double* cov, double* box) {
  std::vector<rec_box_core::Frame> fr(F);
  for (int k = 0; k < F; ++k) {
    const int* v = frames + 7L * k;
    fr[k] = rec_box_core::Frame{v[0], v[1], v[2], v[3], v[4], v[5], v[6]};
  }
  for (long n = 0; n < N; ++n) {
    const long row = n * L;
    int kept = 0;
    for (int j = 0; j < L; ++j) {
      const int kind = rec_box_core::step_kind(rec[row + j], pad, eos);
      if (kind == rec_box_core::kStop) break;
      if (kind == rec_box_core::kSkip) continue;
      const long o = row + kept++;
      step[o] = j;
      rec_box_core::char_box(polys + 32 * n, fr[frame_index[n]], loc + 5 * (row + j), centre + 2 * o, cov + 3 * o,
                             box + 8 * o);
    }
    for (int i = kept; i < L; ++i) {
      const long o = row + i;
      step[o] = 0;
      for (int k = 0; k < 2; ++k) centre[2 * o + k] = 0.0;
      for (int k = 0; k < 3; ++k) cov[3 * o + k] = 0.0;
      for (int k = 0; k < 8; ++k) box[8 * o + k] = 0.0;
    }
    n_chars[n] = kept;
  }
}

// rec_box_core::valid_frame of one frame [7]
int emu_valid_frame(const int* v) {
  return rec_box_core::valid_frame(rec_box_core::Frame{v[0], v[1], v[2], v[3], v[4], v[5], v[6]});
}

}  // extern "C"
