// tests/host_walk/host_walk_kw8.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libabyssb200).
//
// host_walk with the eight-word instance (Kmer<8>) that the kernels use for k = 193..256; k <= 192 goes to host_walk's own
// driver.  Same arguments and environment as host_walk.
#define main host_walk_main
#include "host_walk.cpp"
#undef main

int main(int argc, char** argv)
{
	if (argc >= 7 && (2u * (unsigned)atoi(argv[1]) + 63) / 64 > 6)
		return run<8>(atoi(argv[1]), atoi(argv[2]), atoi(argv[3]), strtoull(argv[4], 0, 10), atoi(argv[5]), argv[6],
		              argc > 7 ? argv[7] : nullptr);
	return host_walk_main(argc, argv);
}
