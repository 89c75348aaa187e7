// BLS12-377 instantiation of the proving engine (377-bit base field in 12 x 32-bit limbs; Fq2 = Fq[u]/(u^2 + 5)).
#include "engine.cuh"
#include "setup.cuh"
#include "gm17.cuh"
namespace zkb {
typedef Engine<CurveT<Bls377Fr, Bls377Fq>> EngineBls377;
EngineBase* make_engine_bls12_377(Stream st) { return new EngineBls377(st); }
size_t partial_bytes_bls12_377() { return sizeof(EngineBls377::Partial); }
}  // namespace zkb
