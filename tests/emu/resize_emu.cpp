// TEST INFRASTRUCTURE — host emulation of programs with CSNET_OP_RESIZE ops (sod100k_b200/csrc/resize.cuh).
//
// Walks a program as plan.cu does: a RESIZE op runs the kernel's per-pixel function (resize_value with mae_tap's taps) over every
// output element; every other op goes, one at a time, through the generic-op emulation of emu.cpp on the same arena and externals.
// fp32 tensors only.
#include "emu.cpp"
#include "../../sod100k_b200/csrc/resize.cuh"

extern "C" int csnet_emu_run_resize(const csnet_tensor_desc* tensors, int n_tensors, const csnet_op_desc* ops, int n_ops,
                                    const float* blob, int N, void* const* ext, char* arena) {
  auto ptr = [&](int t) -> void* {
    const csnet_tensor_desc& d = tensors[t];
    return d.external >= 0 ? ext[d.external] : (void*)(arena + (int64_t)N * d.arena_offset);
  };
  for (int i = 0; i < n_tensors; ++i)
    if (tensors[i].dtype != CSNET_F32) return -4;
  for (int k = 0; k < n_ops; ++k) {
    const csnet_op_desc& op = ops[k];
    if (op.kind != CSNET_OP_RESIZE) {
      const int rc = csnet_emu_run(tensors, n_tensors, ops + k, 1, blob, N, ext, arena);
      if (rc != 0) return rc;
      continue;
    }
    const csnet_tensor_desc& D = tensors[op.dst];
    const csnet_path_desc& q = op.paths[0];
    const csnet_tensor_desc& S = tensors[q.src];
    const float* x = (const float*)ptr(q.src);
    float* y = (float*)ptr(op.dst);
    const bool acc = op.ext_off[0] == 1;
    const float sy = csnet::resize_scale(S.H, D.H), sx = csnet::resize_scale(S.W, D.W);
#pragma omp parallel for collapse(2) schedule(static)
    for (int n = 0; n < N; ++n)
      for (int c = 0; c < q.cout; ++c) {
        const float* plane = x + ((int64_t)n * S.C + q.c0 + c) * S.H * S.W;
        float* out = y + ((int64_t)n * D.C + q.cout0 + c) * D.H * D.W;
        for (int oy = 0; oy < D.H; ++oy)
          for (int ox = 0; ox < D.W; ++ox) {
            float& o = out[(int64_t)oy * D.W + ox];
            o = csnet::resize_value(plane, S.W, csnet::mae_tap(oy, S.H, sy), csnet::mae_tap(ox, S.W, sx), acc, acc ? o : 0.f);
          }
      }
  }
  return 0;
}
