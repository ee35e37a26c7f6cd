// Instantiations of the wide derivative-observation q-KG kernel (9 <= g <= 31) for padded dimension 16 (one translation
// unit per dimension so the build parallelises); registered into the run-time dispatch table of kg.cu.
#include "kg_mc.cuh"

namespace cmoe {
namespace {
const KgDispatchEntry kEntries[] = {CMOE_KG_WIDE_ENTRIES_FOR_DIM(16)};
struct Registrar {
  Registrar() { register_kg_entries(kEntries, static_cast<int>(sizeof(kEntries) / sizeof(kEntries[0]))); }
} registrar;
}  // namespace
}  // namespace cmoe
