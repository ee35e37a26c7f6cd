// Instantiations of the fused q-KG kernels for padded dimension 12 (one translation unit per dimension so the build
// parallelises); registered into the run-time dispatch table of kg.cu.
#include "kg_mc.cuh"

namespace cmoe {
namespace {
const bool registered = register_kg_entries({CMOE_KG_ENTRIES_FOR_DIM(12)});
const bool registered_large = register_kg_large_entries({CMOE_KG_LARGE_ENTRIES_FOR_DIM(12)});
}  // namespace
}  // namespace cmoe
