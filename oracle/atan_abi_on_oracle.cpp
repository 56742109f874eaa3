// atan_abi_on_oracle.cpp — TEST INFRASTRUCTURE ONLY: plsvo_match_direct_atan_batch_run answered by the CPU oracle's ATAN
// matcher (oracle/atan_match_oracle.cpp), next to abi_on_oracle.cpp's pinhole entry points.
//
// Like abi_on_oracle.cpp this is NOT a CPU fallback of the product.  It lets the shim's packing of reference objects whose
// frames hold a vk::ATANCamera (DirectMatcher on ATAN frames) be checked on a machine without a GPU:
// oracle_atan_match.build_shimref(cpu=True) links atan_match_shimref_harness.cpp + the shim + abi_on_oracle.cpp + this file
// + atan_match_oracle.cpp into oracle/_ref/libplsvo_atan_match_shimref_cpu.so.
#include "../include/plsvo_b200.h"

extern "C" {
int plsvo_oracle_atan_match_direct_batch(const plsvo_atan_camera*, const plsvo_match_batch*, const plsvo_match_result*, int);

int plsvo_match_direct_atan_batch_run(plsvo_ctx*, const plsvo_atan_camera* cam, const plsvo_match_batch* b, const plsvo_match_result* o) {
  return plsvo_oracle_atan_match_direct_batch(cam, b, o, 4);
}
}
