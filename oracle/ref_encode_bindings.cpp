// TEST INFRASTRUCTURE (oracle) -- not product code.
//
// pybind11 stub that exposes the reference's trellis encoder (quantize_tiles, pack_trellis: exllamav3_ext/bindings.cpp:116,119)
// from its UNMODIFIED translation units, compiled in place by oracle/build_ref_encode.py into oracle/_ref/exl3_ref_encode.so.
// It only declares/binds functions; all implementations come from the reference's own sources.

#include <torch/extension.h>
#include "quant/quantize.cuh"
#include "quant/pack.cuh"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m)
{
    m.def("quantize_tiles", &quantize_tiles, "quantize_tiles");
    m.def("pack_trellis", &pack_trellis, "pack_trellis");
}
