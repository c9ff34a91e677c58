// Test infrastructure only: oracle/shim/config.h with MAX_KMER = 256 (configure --enable-maxk=256) for the second build of
// the UNMODIFIED reference (oracle/maxk256.mk).  It comes first on the include path, so shim/config.h is never read.
#ifndef CONFIG_H
#define CONFIG_H 1
#define HAVE_STD_HASH 1
#define HAVE_UNORDERED_SET 1
#define HAVE_UNORDERED_MAP 1
#define HAVE_POPCNT 1
#define HAVE_GETOPT_LONG 1
#define HAVE_LIBDL 1
#define MAX_KMER 256
#define MAX_HASHES 32
#define FMBITS 64
#define PACKAGE_NAME "ABySS"
#define PACKAGE_BUGREPORT "abyss-users@bcgsc.ca"
#define VERSION "2.3.10"
#define PACKAGE_STRING "ABySS 2.3.10"
#endif
