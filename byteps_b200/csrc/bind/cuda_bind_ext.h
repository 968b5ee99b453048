// Further kernel families (compression, local optimizers, copies) register
// their bindings from their own translation units.
#pragma once
#include <pybind11/pybind11.h>

void bind_cuda_ext(pybind11::module_& m);
void bind_cuda_ring(pybind11::module_& m);
void bind_cuda_compress(pybind11::module_& m);
void bind_cuda_bn(pybind11::module_& m);
void bind_cuda_ln(pybind11::module_& m);
void bind_cuda_xent(pybind11::module_& m);
void bind_cuda_fp8(pybind11::module_& m);
void bind_cuda_lamb(pybind11::module_& m);
void bind_cuda_lars(pybind11::module_& m);
void bind_cuda_clip(pybind11::module_& m);
void bind_cuda_attn(pybind11::module_& m);
void bind_cuda_mlm(pybind11::module_& m);
void bind_cuda_stem(pybind11::module_& m);
