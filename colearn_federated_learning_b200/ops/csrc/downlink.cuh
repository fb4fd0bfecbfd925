// Downlink compression of the global model: coordinator and devices keep a replica r of the model the devices hold.  Round 0
// of a training sends theta as fp32 (r = theta); every later round the coordinator encodes v = theta - r ONCE, broadcasts the
// same bytes to every device, and both sides advance r by what was sent, bit for bit alike.  Whatever has not been delivered
// yet is theta - r: it stays on the coordinator and goes out in later rounds (error feedback with no residual array).
// downlink_quant_kernel / downlink_topk_kernel (encode and advance, coordinator) and replica_apply_q_kernel /
// replica_apply_topk_kernel (advance from the wire, device) in elementwise.cu use these functions; the GPU build and the SIMT
// CPU build (host_shim.h) both compile them, and ops/reference.py encode_downlink / apply_downlink is the numpy transcription.
//
// The codecs are the uplink's, with the same wire layout:
//   int8 / int4 (uplink_quant.cuh): the codes and block steps of d = theta - r (one fp32 subtraction) with one key per round
//                shared by every device; then r_j <- r_j + uq_decode(q_j, step) (one fp32 add, written dl_add_rn so that it
//                cannot contract with the decode's product into an FMA).  A block of step 0 adds +0 (r = -0 becomes +0).
//   topk       (uplink_topk.cuh): v_j = theta_j - r_j (the only subtraction), the selection and wire of the uplink with no
//                residual input; then r_j <- r_j + v_j for the sent entries, nothing else changes.
// A non-finite v / d reaches the wire (NaN step, or a non-finite value) and the replica; devices refuse such a wire.
// Included by colearn_kernels.h after uplink_topk.cuh.
#pragma once

namespace colearn {

COLEARN_HD float dl_add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// the replica after the int8 / int4 code q of step `step` arrived
COLEARN_HD float dl_quant_advance(float r, int q, float step) { return dl_add_rn(r, uq_decode(q, step)); }

}  // namespace colearn
