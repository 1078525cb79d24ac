// TEST INFRASTRUCTURE (oracle) -- not product code.
//
// pybind11 stub that exposes the reference's RMSNorm operators (rms_norm, rms_norm_res_in, gated_rms_norm:
// exllamav3_ext/bindings.cpp:84-86) from its UNMODIFIED norm.cu, compiled in place by oracle/build_ref_norm.py into
// oracle/_ref/exl3_ref_norm.so.  It only declares/binds functions; all implementations come from the reference's own sources.

#include <torch/extension.h>
#include "norm.cuh"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m)
{
    m.def("rms_norm", &rms_norm, "rms_norm");
    m.def("rms_norm_res_in", &rms_norm_res_in, "rms_norm_res_in");
    m.def("gated_rms_norm", &gated_rms_norm, "gated_rms_norm");
}
