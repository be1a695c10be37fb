// ffma_inst.cu -- one explicit instantiation of the fused kernel per translation unit
// (compiled 24 times: {float,double} x {activation buffers in smem, in global} x {plain, with integral terms, with
// fixed networks (and integral terms), with a functional term (and both)}, and the double ones again with the layer
// products on DMMA (PINN_MODE_TC_F64)) so the build parallelises.
// -DPINN_INST_REAL=float|double -DPINN_INST_BUFS=0|1 [-DPINN_INST_INTEG=1 [-DPINN_INST_FIXED=1 [-DPINN_INST_FUNC=1]]]
// [-DPINN_INST_DMMA=1]
#include "ffma_kernel.cuh"

namespace pinn {

#define PINN_CAT2(a, b) a##b
#define PINN_CAT(a, b) PINN_CAT2(a, b)
#if PINN_INST_BUFS
#define PINN_BUFS_NAME smem
#else
#define PINN_BUFS_NAME gmem
#endif
#ifndef PINN_INST_INTEG
#define PINN_INST_INTEG 0
#endif
#ifndef PINN_INST_FIXED
#define PINN_INST_FIXED 0
#endif
#ifndef PINN_INST_FUNC
#define PINN_INST_FUNC 0
#endif
#ifndef PINN_INST_DMMA
#define PINN_INST_DMMA 0
#endif
#if PINN_INST_FUNC
#define PINN_BUFS_NAME_X PINN_CAT(PINN_BUFS_NAME, _func)
#elif PINN_INST_FIXED
#define PINN_BUFS_NAME_X PINN_CAT(PINN_BUFS_NAME, _fixed)
#elif PINN_INST_INTEG
#define PINN_BUFS_NAME_X PINN_CAT(PINN_BUFS_NAME, _integ)
#else
#define PINN_BUFS_NAME_X PINN_BUFS_NAME
#endif
#if PINN_INST_DMMA
#define PINN_LAUNCH_NAME PINN_CAT(PINN_CAT(PINN_CAT(ffma_launch_, PINN_INST_REAL), _dmma_), PINN_BUFS_NAME_X)
#else
#define PINN_LAUNCH_NAME PINN_CAT(PINN_CAT(PINN_CAT(ffma_launch_, PINN_INST_REAL), _), PINN_BUFS_NAME_X)
#endif

cudaError_t PINN_LAUNCH_NAME(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st) {
  return launch_fused_kernel<ffma_loss_grad_kernel<PINN_INST_REAL, (PINN_INST_BUFS != 0), (PINN_INST_INTEG != 0),
                                                   (PINN_INST_FIXED != 0), (PINN_INST_FUNC != 0), (PINN_INST_DMMA != 0)>>(
      a, grid, kThreads, smem, st);
}

}  // namespace pinn
