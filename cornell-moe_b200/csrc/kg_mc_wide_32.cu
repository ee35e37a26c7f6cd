// Instantiations of the wide derivative-observation q-KG kernel (9 <= g <= 31) for padded dimension 32 (one translation
// unit per dimension so the build parallelises); registered into the run-time dispatch table of kg.cu.
#include "kg_mc.cuh"

namespace cmoe {
namespace {
const bool registered = register_kg_entries({CMOE_KG_WIDE_ENTRIES_FOR_DIM(32)});
const bool registered_large = register_kg_large_entries({CMOE_KG_LARGE_WIDE_ENTRIES_FOR_DIM(32)});
}  // namespace
}  // namespace cmoe
