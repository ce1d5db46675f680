// poa_trace_kernel.cu -- the trace kernels poa_trace_kernel_t* (barb200_poa_trace_batch): poa_kernel.cu's kernel body with
// TRACE = true, which also appends every alignment's record to the job's trace region (poa_kernel.cu: trace_record). A module of its
// own, so that the production kernels' module (poa_kernel.cu) holds only them and compiles to the code it has without trace kernels.
//
// Both objects go into one library and both define the non-inline functions of the kernel's headers, so this module's copies are
// renamed: every `barb200` namespace of the product's headers becomes barb200_trace_module here (no system header names it). The
// kernels are extern "C": their names, which barb200.cu declares, do not change.
#define BARB200_TRACE_KERNELS
#define barb200 barb200_trace_module
#include "poa_kernel.cu"
