"""The reference's python binding surface for the conv library, on libconvnet_b200.so.

Same function names and argument meaning as cudamat/cudamat_conv_gemm.py:61-157
(`convUp(images, filters, targets, conv_desc, scaleTargets=0)` ...) and
cudamat/cudamat_conv.py for the second symbol set, so the parity tests read like
py/test_conv.py.  Arguments are CUDAMatrix objects.

`Binding(get_lib, abi)` is the surface bound to one shared library and one symbol set:
  abi = "gemm": ABI-1, the `*Gemm` names of cudamat_conv_gemm.cuh:36-138 (default build of the reference)
  abi = "cc2" : ABI-2, the bare names of cudamat_conv.cuh:8-78 (pool forward has no scale arguments,
                ResponseNormCrossMapUndo takes `acts`, convOutp takes the partial-sum sizes)
The module-level functions are `Binding(lib.load, "gemm")`; `cc2` is the ABI-2 twin.  A test may bind the same
surface to another library that exports these symbols (the reference's own CUDA build, tests/ref_cuda_lib.py).
"""
from . import lib as _lib


class Binding:
    def __init__(self, get_lib, abi="gemm"):
        assert abi in ("gemm", "cc2")
        self._get, self.abi = get_lib, abi
        self._sfx = "Gemm" if abi == "gemm" else ""

    def _f(self, name):
        return getattr(self._get(), name + self._sfx)

    # ---- convolution ----------------------------------------------------------------------------
    def convUp(self, images, filters, targets, conv_desc, scaleTargets=0):
        self._f("convUp")(images.p_mat, filters.p_mat, targets.p_mat, images.p_shape4d, filters.p_shape4d,
                          targets.p_shape4d, conv_desc, scaleTargets)

    def convDown(self, hidSums, filters, targets, conv_desc, scaleTargets=0):
        self._f("convDown")(hidSums.p_mat, filters.p_mat, targets.p_mat, hidSums.p_shape4d, filters.p_shape4d,
                            targets.p_shape4d, conv_desc, scaleTargets)

    def convOutp(self, images, hidSums, targets, conv_desc, scaleTargets=0, scaleGradients=1):
        if self.abi == "cc2":      # partialSum 0/0 = one sum over all modules (cudamat_conv.py convOutp)
            return self.convOutpPartial(images, hidSums, targets, conv_desc, 0, 0, scaleTargets, scaleGradients)
        self._f("convOutp")(images.p_mat, hidSums.p_mat, targets.p_mat, images.p_shape4d, hidSums.p_shape4d,
                            targets.p_shape4d, conv_desc, scaleTargets, scaleGradients)

    def convOutpPartial(self, images, hidSums, targets, conv_desc, partialSumY, partialSumX, scaleTargets=0,
                        scaleGradients=1):
        """ABI-2 only (cudamat_conv.cuh:26-29)."""
        self._get().convOutp(images.p_mat, hidSums.p_mat, targets.p_mat, images.p_shape4d, hidSums.p_shape4d,
                             targets.p_shape4d, conv_desc, partialSumY, partialSumX, scaleTargets, scaleGradients)

    def convInnerp(self, images, hidSums, targets, conv_desc, scaleTargets=0, scaleGradients=1):
        """ABI-1 only (cudamat_conv_gemm.py convInnerp): targets, shape (1, kx, ky, 1), gets per filter tap the sum over
        images, modules and channels of the image patch value times the derivative of the same channel"""
        self._get().convInnerpGemm(images.p_mat, hidSums.p_mat, targets.p_mat, images.p_shape4d, hidSums.p_shape4d,
                                   targets.p_shape4d, conv_desc, scaleTargets, scaleGradients)

    def localUp(self, images, filters, targets, conv_desc, scaleTargets=0):
        self._f("localUp")(images.p_mat, filters.p_mat, targets.p_mat, images.p_shape4d, filters.p_shape4d,
                           targets.p_shape4d, conv_desc, scaleTargets)

    def localDown(self, hidSums, filters, targets, conv_desc, scaleTargets=0):
        self._f("localDown")(hidSums.p_mat, filters.p_mat, targets.p_mat, hidSums.p_shape4d, filters.p_shape4d,
                             targets.p_shape4d, conv_desc, scaleTargets)

    def localOutp(self, images, hidSums, targets, conv_desc, scaleTargets=0, scaleGradients=1):
        self._f("localOutp")(images.p_mat, hidSums.p_mat, targets.p_mat, images.p_shape4d, hidSums.p_shape4d,
                             targets.p_shape4d, conv_desc, scaleTargets, scaleGradients)

    # ---- pooling ----------------------------------------------------------------------------------
    def MaxPool(self, images, targets, conv_desc):
        extra = (0.0, 1.0) if self.abi == "gemm" else ()
        self._f("MaxPool")(images.p_mat, targets.p_mat, images.p_shape4d, targets.p_shape4d, conv_desc, *extra)

    def MaxPoolRprop(self, images, R_images, maxes, targets, conv_desc, scaleTargets=0):
        """ABI-1 only (cudamat_conv_gemm.py MaxPoolRprop): the R-operator of max pooling"""
        self._get().MaxPoolRpropGemm(images.p_mat, R_images.p_mat, maxes.p_mat, targets.p_mat, images.p_shape4d,
                                     maxes.p_shape4d, conv_desc, scaleTargets)

    def AvgPool(self, images, targets, conv_desc):
        extra = (0.0, 1.0) if self.abi == "gemm" else ()
        self._f("AvgPool")(images.p_mat, targets.p_mat, images.p_shape4d, targets.p_shape4d, conv_desc, *extra)

    def MaxPoolUndo(self, images, grad, maxes, targets, conv_desc, scaleTargets=0):
        self._f("MaxPoolUndo")(images.p_mat, grad.p_mat, maxes.p_mat, targets.p_mat, images.p_shape4d,
                               grad.p_shape4d, conv_desc, scaleTargets)

    def AvgPoolUndo(self, avgGrads, targets, conv_desc, scaleTargets=0):
        self._f("AvgPoolUndo")(avgGrads.p_mat, targets.p_mat, avgGrads.p_shape4d, targets.p_shape4d, conv_desc,
                               scaleTargets)

    def UpSample(self, images, targets, factor, scaleTargets=0):
        self._f("UpSample")(images.p_mat, targets.p_mat, images.p_shape4d, targets.p_shape4d, factor, scaleTargets)

    def DownSample(self, images, targets, factor):
        self._f("DownSample")(images.p_mat, targets.p_mat, images.p_shape4d, targets.p_shape4d, factor)

    # ---- cross-map response normalisation -------------------------------------------------------------
    def ResponseNormCrossMap(self, images, targets, sizeF, addScale, powScale, blocked):
        num_filters = images.shape4d[3]
        self._f("ResponseNormCrossMap")(images.p_mat, targets.p_mat, num_filters, sizeF, addScale, powScale, blocked)

    def ResponseNormCrossMapUndo(self, derivs, images, targets, sizeF, addScale, powScale, blocked, acts=None):
        num_filters = images.shape4d[3]
        if self.abi == "cc2":      # cudamat_conv.cuh:39-42: (outGrads, inputs, acts, targets, ...)
            acts = acts if acts is not None else images
            self._f("ResponseNormCrossMapUndo")(derivs.p_mat, images.p_mat, acts.p_mat, targets.p_mat, num_filters,
                                                sizeF, addScale, powScale, blocked)
        else:
            self._f("ResponseNormCrossMapUndo")(derivs.p_mat, images.p_mat, targets.p_mat, num_filters, sizeF,
                                                addScale, powScale, blocked)

    def ResponseNormCrossMapRprop(self, images, R_images, targets, sizeF, addScale, powScale, blocked):
        """ABI-1 only (cudamat_conv_gemm.py ResponseNormCrossMapRprop): the R-operator of cross-map normalisation"""
        num_filters = images.shape4d[3]
        self._get().ResponseNormCrossMapRpropGemm(images.p_mat, R_images.p_mat, targets.p_mat, num_filters, sizeF,
                                                  addScale, powScale, blocked)

    # ---- within-map normalisation and colour (ABI-2 only: cudamat_conv.cuh:44-78) -------------------------------------
    def ResponseNorm(self, images, denoms, targets, numChannels, sizeX, addScale, powScale):
        self._get().ResponseNorm(images.p_mat, denoms.p_mat, targets.p_mat, numChannels, sizeX, addScale, powScale)

    def ResponseNormUndo(self, outGrad, denoms, inGrad, acts, targets, numChannels, sizeX, addScale, powScale):
        self._get().ResponseNormUndo(outGrad.p_mat, denoms.p_mat, inGrad.p_mat, acts.p_mat, targets.p_mat, numChannels,
                                     sizeX, addScale, powScale)

    def ContrastNorm(self, images, meanDiffs, denoms, targets, numChannels, sizeX, addScale, powScale):
        self._get().ContrastNorm(images.p_mat, meanDiffs.p_mat, denoms.p_mat, targets.p_mat, numChannels, sizeX,
                                 addScale, powScale)

    def ContrastNormUndo(self, outGrad, denoms, meanDiffs, acts, targets, numChannels, sizeX, addScale, powScale):
        self._get().ContrastNormUndo(outGrad.p_mat, denoms.p_mat, meanDiffs.p_mat, acts.p_mat, targets.p_mat,
                                     numChannels, sizeX, addScale, powScale)

    def RGBToYUV(self, images, targets):
        """images: (numImages, 3 * pixels), the R, G and B planes; targets: the Y, U and V planes, same shape"""
        self._get().RGBToYUV(images.p_mat, targets.p_mat)

    # ---- 3-D (ABI-1 only: cudamat_conv3d_gemm.cu) -----------------------------------------------------
    def ResponseNormCrossMap3D(self, images, targets, sizeF, addScale, powScale, blocked, image_size_t):
        num_filters = images.shape4d[3] // image_size_t
        self._get().ResponseNormCrossMap3DGemm(images.p_mat, targets.p_mat, num_filters, sizeF, addScale, powScale,
                                               blocked, image_size_t)

    def ResponseNormCrossMap3DUndo(self, derivs, images, targets, sizeF, addScale, powScale, blocked, image_size_t):
        num_filters = images.shape4d[3] // image_size_t
        self._get().ResponseNormCrossMap3DUndoGemm(derivs.p_mat, images.p_mat, targets.p_mat, num_filters, sizeF,
                                                   addScale, powScale, blocked, image_size_t)

    def convUp3D(self, images, filters, targets, conv_desc, scaleTargets=0):
        self._get().convUp3DGemm(images.p_mat, filters.p_mat, targets.p_mat, images.p_shape4d, filters.p_shape4d,
                                 targets.p_shape4d, conv_desc, scaleTargets)

    def convDown3D(self, hidSums, filters, targets, conv_desc, scaleTargets=0):
        self._get().convDown3DGemm(hidSums.p_mat, filters.p_mat, targets.p_mat, hidSums.p_shape4d,
                                   filters.p_shape4d, targets.p_shape4d, conv_desc, scaleTargets)

    def convOutp3D(self, images, hidSums, targets, conv_desc, scaleTargets=0, scaleGradients=1):
        self._get().convOutp3DGemm(images.p_mat, hidSums.p_mat, targets.p_mat, images.p_shape4d, hidSums.p_shape4d,
                                   targets.p_shape4d, conv_desc, scaleTargets, scaleGradients)

    # 3-D pooling goes through the same entry points (kernel_size_t/stride_t in the descriptor)
    def MaxPool3D(self, *a, **k): return self.MaxPool(*a, **k)
    def MaxPool3DUndo(self, *a, **k): return self.MaxPoolUndo(*a, **k)
    def AvgPool3D(self, *a, **k): return self.AvgPool(*a, **k)
    def AvgPool3DUndo(self, *a, **k): return self.AvgPoolUndo(*a, **k)

    def SetupTexture(self, mat):
        """ABI-2 only (cudamat_conv.cuh:8)."""
        self._get().SetupTexture(mat.p_mat)


gemm = Binding(_lib.load, "gemm")      # ABI-1 on libconvnet_b200.so
cc2 = Binding(_lib.load, "cc2")        # ABI-2 on libconvnet_b200.so

# module-level ABI-1 functions, the names cudamat_conv_gemm.py exports
convUp, convDown, convOutp = gemm.convUp, gemm.convDown, gemm.convOutp
localUp, localDown, localOutp = gemm.localUp, gemm.localDown, gemm.localOutp
MaxPool, AvgPool, MaxPoolUndo, AvgPoolUndo = gemm.MaxPool, gemm.AvgPool, gemm.MaxPoolUndo, gemm.AvgPoolUndo
UpSample, DownSample = gemm.UpSample, gemm.DownSample
ResponseNormCrossMap, ResponseNormCrossMapUndo = gemm.ResponseNormCrossMap, gemm.ResponseNormCrossMapUndo
ResponseNormCrossMap3D, ResponseNormCrossMap3DUndo = gemm.ResponseNormCrossMap3D, gemm.ResponseNormCrossMap3DUndo
convUp3D, convDown3D, convOutp3D = gemm.convUp3D, gemm.convDown3D, gemm.convOutp3D
MaxPool3D, MaxPool3DUndo, AvgPool3D, AvgPool3DUndo = MaxPool, MaxPoolUndo, AvgPool, AvgPoolUndo
convOutpPartial = gemm.convOutpPartial
convInnerp, MaxPoolRprop, ResponseNormCrossMapRprop = gemm.convInnerp, gemm.MaxPoolRprop, gemm.ResponseNormCrossMapRprop
ResponseNorm, ResponseNormUndo, ContrastNorm, ContrastNormUndo = cc2.ResponseNorm, cc2.ResponseNormUndo, cc2.ContrastNorm, cc2.ContrastNormUndo
RGBToYUV = cc2.RGBToYUV
