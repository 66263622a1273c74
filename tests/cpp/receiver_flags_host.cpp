// receiver_flags_host.cpp -- TEST HARNESS: compiles the receiver flags table's word rules (libcimbar_b200/csrc/receivers_core.cuh:
// word_refused, word_sharpens, word_passes) for the host, so that they can be checked against a restatement where there is no GPU.
// Not part of the product; the product runs the same functions in k_extract and k_ccm_carry_receivers.
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

using namespace cb200::receivers;

// per word: bit 0 refused, bit 1 sharpened at extract status 2, bit 2 sharpened at status 1, bit 3 passes its CCM through in a mode
// that fits, bit 4 passes it through in a mode that never fits
extern "C" void rf_rules(const uint32_t* words, int n, uint8_t* out)
{
    for (int i = 0; i < n; ++i) {
        const uint32_t w = words[i];
        out[i] = (uint8_t)((word_refused(w) ? 1 : 0) | (word_sharpens(w, 2) ? 2 : 0) | (word_sharpens(w, 1) ? 4 : 0) |
                           (word_passes(w, true) ? 8 : 0) | (word_passes(w, false) ? 16 : 0));
    }
}
