# oracle/maxk256.mk -- TEST INFRASTRUCTURE ONLY.
#
# The UNMODIFIED reference built a second time with MAX_KMER = 256 (configure --enable-maxk=256): the oracle of k = 193..256
# (tests/golden/make_golden_kwidth256.py).  Makefile's rules and sources, with shim_maxk256/ (config.h with MAX_KMER 256)
# ahead of shim/ on the include path, into oracle/_ref/maxk256/.
#
#   make -C oracle -f maxk256.mk REF=...   # needs a source tree of the reference, as `make -C oracle ref` does

REF ?= $(abspath $(CURDIR)/../../reference)
OUT := _ref/maxk256
RF  := -std=c++11 -O2 -fopenmp -w -include getopt.h -Ishim_maxk256 -Ishim -I$(REF) -I$(REF)/Common -I$(REF)/DataLayer -I$(REF)/vendor

.PHONY: maxk256
maxk256:
	$(MAKE) -f Makefile check-ref $(OUT)/abyss-bloom-dbg-ref $(OUT)/abyss-bloom-ref $(OUT)/AdjList-ref OUT=$(OUT) RF="$(RF)" REF=$(REF)
