// Hidden-layer activation of the neural-network coupling layer (B2B_COUPLING_MLP), shared by its forward and
// reverse-mode kernels: h = σ(v) and σ′(v).
#pragma once
#include "b2b_device.cuh"

namespace b2b {

// B2B_ACT_TANH: tanh and sech² from one exponential (tanh_sech2).  B2B_ACT_LEAKY_RELU: v >= 0 ? v : a·v
// (leaky_relu.jl:18-29), so σ′(0) = 1.
__device__ __forceinline__ void mlp_act(int act, float slope, float v, float& h, float& dh) {
  if (act == B2B_ACT_TANH) {
    tanh_sech2(v, h, dh);
  } else {
    dh = v >= 0.f ? 1.0f : slope;
    h = v >= 0.f ? v : slope * v;
  }
}

}  // namespace b2b
