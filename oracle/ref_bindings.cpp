// TEST INFRASTRUCTURE (oracle) -- not product code.
//
// pybind11 stub that exposes the hot-path subset of the UNMODIFIED reference extension
// (exllamav3/exllamav3_ext of the checkout named by $EXLLAMAV3_SOURCE, compiled in place by oracle/build_ref.py into oracle/_ref/).
// It only declares/binds functions; all implementations come from the reference's own translation units.
// The reference's bindings.cpp binds its whole ~150-TU extension; this binds what the EXL3 qgemm path needs
// (reference bindings: exllamav3_ext/bindings.cpp:118-147).

#include <torch/extension.h>
#include "quant/exl3_gemm.cuh"
#include "quant/reconstruct.cuh"
#include "quant/hadamard.cuh"
#include "hgemm.cuh"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m)
{
    m.def("exl3_gemm", &exl3_gemm, "exl3_gemm");
    m.def("exl3_mgemm", &exl3_mgemm, "exl3_mgemm",
          py::arg("A"), py::arg("B"), py::arg("C"), py::arg("suh"), py::arg("A_had"), py::arg("svh"),
          py::arg("indices"), py::arg("weights"), py::arg("K"), py::arg("force_shape_idx"),
          py::arg("mcg_mult"), py::arg("mul1_mult"), py::arg("min_index"), py::arg("max_index"),
          py::arg("force_num_sms"), py::arg("num_tokens") = 1,
          py::arg("size_n_list") = py::none(), py::arg("c_ptrs") = py::none());
    m.def("reconstruct", &reconstruct, "reconstruct");
    m.def("reconstruct_slice", &reconstruct_slice, "reconstruct_slice");
    m.def("reconstruct_had_slice", &reconstruct_had_slice, "reconstruct_had_slice");
    m.def("had_r_128", &had_r_128, "had_r_128");
    m.def("hgemm", &hgemm, "hgemm");
}
