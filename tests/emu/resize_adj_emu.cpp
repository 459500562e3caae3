// TEST INFRASTRUCTURE — the resize adjoint's tap inversion (sod100k_b200/csrc/resize_adj.cuh) compiled for the CPU.
#define CSNET_HOST_EMU
#include "../../sod100k_b200/csrc/resize_adj.cuh"

// adj[s * n_out + o] = the weight source s receives from output o along one axis of n_in -> n_out samples, as the backward gathers it.
extern "C" void csnet_emu_resize_adjoint(int n_in, int n_out, double* adj) {
  const float scale = csnet::resize_scale(n_in, n_out);
  for (int s = 0; s < n_in; ++s) {
    for (int o = 0; o < n_out; ++o) adj[(long)s * n_out + o] = 0.0;
    const csnet::RzRange r = csnet::rz_src_range(s, n_in, n_out, scale);
    for (int o = r.lo; o <= r.hi; ++o) adj[(long)s * n_out + o] = csnet::rz_adj_weight(csnet::mae_tap(o, n_in, scale), s);
  }
}
