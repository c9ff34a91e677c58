// tests/host_trim/host_trim_kw8.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// host_trim over the eight-word Konnector k-mer (KonKmerN<8>) that k_kon_trim uses for k = 193..256.  Same arguments as
// host_trim.
#include "../../abyss_b200/csrc/abb_konnector.cuh"
#define KonVtx KonVtxN<kKonWordsWide>
#define kon_left_trim kon_left_trim<kKonWordsWide>
#include "host_trim.cpp"
