// abb_device.cuh -- arithmetic shared by all kernels: closed-form ntHash, multi-hash, exact
// 64-bit modulo by an invariant divisor, 2-bit base codes.
//
// ntHash (reference: vendor/nthash/nthash.hpp:196-342) is linear over XOR: with R = "rotate the
// low 33 bits and the high 31 bits left by one, each inside its own field" (rol1+swapbits033,
// :196-211), the forward hash of a k-mer c_0..c_{k-1} is XOR_i R^{k-1-i}(seed(c_i)) and the
// reverse-complement hash is XOR_i R^{i}(seed(comp c_i)) (:220-239).  R has period 33*31 = 1023,
// so R^n for any n is two field rotations by n%33 and n%31 -- that is what the msTab31l/msTab33r
// tables hold (:66-194).  Nothing here is sequential; the kernels evaluate it per position.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ABB_HD __host__ __device__ __forceinline__
#define ABB_D __device__ __forceinline__
#define ABB_HD_NOINLINE __host__ __device__ __noinline__ // rarely taken slow paths: one copy, not one per call site
#else
#define ABB_HD inline
#define ABB_D inline
#define ABB_HD_NOINLINE __attribute__((noinline))
#endif

namespace abb {

constexpr uint64_t kSeedA = 0x3c8bfbb395c60474ULL; // nthash.hpp:25
constexpr uint64_t kSeedC = 0x3193c18562a02b4cULL; // :26
constexpr uint64_t kSeedG = 0x20323ed082572324ULL; // :27
constexpr uint64_t kSeedT = 0x295549f54be24456ULL; // :28
constexpr uint64_t kMultiSeed = 0x90b45d39fb6da1faULL; // :22
constexpr unsigned kMultiShift = 27;                   // :19
constexpr unsigned kMaxHashes = 32;                    // configure.ac:151-159 MAX_HASHES
constexpr unsigned kMaxK = 256;                        // the largest k the kernels are built for (configure --enable-maxk=256)
constexpr unsigned kDefaultMaxK = 192;                 // configure.ac MAX_KMER default: the k accepted until abb_set_max_kmer

constexpr uint64_t kMask33 = 0x1FFFFFFFFULL;
constexpr uint64_t kMask31 = 0x7FFFFFFFULL;

/** 2-bit code of a base (A,C,G,T -> 0..3, either case), 4 for anything else. */
ABB_HD unsigned base_code(unsigned char c)
{
	unsigned u = c & 0xDFu; // fold case (RollingHashIterator.h:131)
	unsigned code = (u >> 1) & 3u;
	code ^= code >> 1; // A=0 C=1 T=2 G=3  ->  A=0 C=1 G=2 T=3
	bool ok = (u == 'A') | (u == 'C') | (u == 'G') | (u == 'T');
	return ok ? code : 4u;
}

/** seed of a 2-bit code; code 4 (non-ACGT) hashes as 0 like seedTab['N'] (nthash.hpp:29,40). */
#if defined(__CUDACC__)
static __device__ __constant__ uint64_t kSeedTabDev[8] = { kSeedA, kSeedC, kSeedG, kSeedT, 0, 0, 0, 0 };
#endif
ABB_HD uint64_t seed_of(unsigned code)
{
#if defined(__CUDA_ARCH__)
	return kSeedTabDev[code & 7]; // constant-bank lookup: one LDC instead of a chain of 64-bit selects
#else
	return code == 0 ? kSeedA : code == 1 ? kSeedC : code == 2 ? kSeedG : code == 3 ? kSeedT : 0ULL;
#endif
}

/** R^n with n given as (n % 33, n % 31). */
ABB_HD uint64_t srol_ab(uint64_t x, unsigned a, unsigned b)
{
	uint64_t lo = x & kMask33, hi = x >> 33;
	lo = ((lo << a) | (lo >> (33 - a))) & kMask33;
	hi = ((hi << b) | (hi >> (31 - b))) & kMask31;
	return (hi << 33) | lo;
}
ABB_HD uint64_t srol_n(uint64_t x, unsigned n) { return srol_ab(x, n % 33u, n % 31u); }
/** R^{-n} */
ABB_HD uint64_t sror_n(uint64_t x, unsigned n)
{
	unsigned a = n % 33u, b = n % 31u;
	return srol_ab(x, a ? 33u - a : 0u, b ? 31u - b : 0u);
}
/** R^1 (nthash.hpp:196-198,208-211) */
ABB_HD uint64_t srol1(uint64_t v)
{
	uint64_t r = (v << 1) | (v >> 63);
	uint64_t x = (r ^ (r >> 33)) & 1;
	return r ^ (x | (x << 33));
}
/** R^-1 (nthash.hpp:201-203,214-217) */
ABB_HD uint64_t sror1(uint64_t v)
{
	uint64_t r = (v >> 1) | (v << 63);
	uint64_t x = ((r >> 32) ^ (r >> 63)) & 1;
	return r ^ ((x << 32) | (x << 63));
}

/** Per-k constants for O(1) rolls: R^k(seed(c)) for c = A,C,G,T (msTab*[c][k%31|k%33]). */
struct RollTab {
	uint64_t rk[4];
	// spaced seed (MaskedKmer::mask(), Common/MaskedKmer.h:22-60): the don't-care positions of the k-mer, ascending,
	// none of them 0 or k-1, in memory the code using the table can read; nmask == 0 when there is no mask
	unsigned nmask;
	const uint8_t* mpos;
};
ABB_HD RollTab make_rolltab(unsigned k)
{
	RollTab t;
	for (unsigned c = 0; c < 4; ++c)
		t.rk[c] = srol_n(seed_of(c), k);
	t.nmask = 0;
	t.mpos = nullptr;
	return t;
}

/** forward / reverse-complement hash state of one k-mer (RollingHash m_hash1 / m_rcHash1) */
struct HashPair {
	uint64_t fh, rh;
	ABB_HD uint64_t canonical() const { return rh < fh ? rh : fh; } // RollingHash.h:28-31
};

/** slide right: drop code `out` on the left, append `in` on the right (nthash.hpp:242-257) */
ABB_HD HashPair roll_right(HashPair h, const RollTab& t, unsigned out, unsigned in)
{
	HashPair r;
	r.fh = srol1(h.fh) ^ seed_of(in) ^ t.rk[out];
	r.rh = sror1(h.rh ^ t.rk[3 - in] ^ seed_of(3 - out));
	return r;
}
/** slide left: drop `out` on the right, prepend `in` on the left (nthash.hpp:282-297) */
ABB_HD HashPair roll_left(HashPair h, const RollTab& t, unsigned out, unsigned in)
{
	HashPair r;
	r.fh = sror1(h.fh ^ t.rk[in] ^ seed_of(out));
	r.rh = srol1(h.rh) ^ seed_of(3 - in) ^ t.rk[3 - out];
	return r;
}

// ---- exact n % d for an invariant 64-bit divisor d ------------------------------------------
// m = floor(2^64 / d) (d >= 2).  q = floor(n * m / 2^64) is floor(n / d) or one less (n * m / 2^64 > n / d - 1 because
// n < 2^64 and 2^64 - m * d < d), so r = n - q * d lies in [0, 2d) and one conditional subtraction makes it exact.
// One 64x64 high multiply + one low multiply (round 1 used a 128-bit reciprocal: two high multiplies + carries);
// this is the inner loop of every Bloom probe.  tests/test_host_arith.py checks it against % on random and adversarial values.
struct FastMod {
	uint64_t d, m_hi, m_lo; // m_hi = floor(2^64 / d); m_lo unused (kept for layout compatibility)
};

#if defined(__CUDA_ARCH__)
ABB_D uint64_t mulhi64(uint64_t a, uint64_t b) { return __umul64hi(a, b); }
#else
inline uint64_t mulhi64(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
#endif

ABB_HD uint64_t fastmod_u64(uint64_t n, const FastMod& f)
{
	const uint64_t q = mulhi64(n, f.m_hi);
	const uint64_t r = n - q * f.d;
	return r >= f.d ? r - f.d : r;
}

inline FastMod make_fastmod(uint64_t d) // host only
{
	FastMod f;
	f.d = d;
	f.m_hi = (uint64_t)((((unsigned __int128)1) << 64) / d); // d >= 2
	f.m_lo = 0;
	return f;
}

/** Everything a kernel needs to turn h0 into H filter positions
 *  (RollingHash::getHashes RollingHash.h:143-148 + `hash % size`, CountingBloomFilter.hpp:57-60). */
struct HashCfg {
	unsigned H, k;
	FastMod mod;               // divisor = number of counters / bits
	uint64_t mult[kMaxHashes]; // i ^ (k * multiSeed), nthash.hpp:339 (C precedence)
};

ABB_HD uint64_t nth_hash(uint64_t h0, const HashCfg& cfg, unsigned i)
{
	if (i == 0)
		return h0;
	uint64_t t = h0 * cfg.mult[i];
	return t ^ (t >> kMultiShift);
}
ABB_HD uint64_t nth_pos(uint64_t h0, const HashCfg& cfg, unsigned i) { return fastmod_u64(nth_hash(h0, cfg, i), cfg.mod); }

} // namespace abb
