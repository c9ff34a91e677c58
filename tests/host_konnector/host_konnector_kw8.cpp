// tests/host_konnector/host_konnector_kw8.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// host_konnector over the eight-word Konnector k-mer (KonKmerN<8>) that k_kon_walk uses for k = 193..256.  Same arguments as
// host_konnector.
#include "../../abyss_b200/csrc/abb_konnector.cuh"
#define KonKmer KonKmerN<kKonWordsWide>
#include "host_konnector.cpp"
