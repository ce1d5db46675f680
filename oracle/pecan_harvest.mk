# oracle/pecan_harvest.mk -- the cPecan-mode recorder build, on top of oracle/Makefile's variables and reference objects (run after
# it: make -C oracle -f pecan_harvest.mk):
#
#   _ref/libflower_pecan_harvest.so  the UNMODIFIED reference flower stack of libflower_ref.so with shim/cactus_pecan_harvest.c
#                                    recording every pair cPecan's multiple aligner aligns (BARB200_PECAN_HARVEST=<file>), for
#                                    replay by scripts/pecan_replay.py. pairwiseAligner.o and multipleAligner.o are linked twice:
#                                    with getAlignedPairs / makeAlignment weakened (callers reach the wrappers) and as private
#                                    ref_-prefixed copies (the wrappers forward to them). Only built where the reference sources exist.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := pecan_harvest
.PHONY: pecan_harvest

ifneq ($(wildcard $(ABPOA)/src/abpoa_align.c),)
pecan_harvest: $(REFDIR)/libflower_pecan_harvest.so
else
pecan_harvest:
	@echo "oracle/pecan_harvest.mk: $(REFERENCE) not present; keeping prebuilt oracle/_ref (if any)"
endif

$(REFDIR)/obj/pecan/pairwiseAligner_hweak.o: $(REFDIR)/obj/pecan/pairwiseAligner.o
	@objcopy --weaken-symbol=getAlignedPairs $< $@
$(REFDIR)/obj/pecan/multipleAligner_hweak.o: $(REFDIR)/obj/pecan/multipleAligner.o
	@objcopy --weaken-symbol=makeAlignment $< $@
$(REFDIR)/obj/pecan/%_private.o: $(REFDIR)/obj/pecan/%.o
	@nm -g --defined-only $< | awk '{print $$3 " ref_" $$3}' > $(REFDIR)/obj/pecan/$*_syms.txt
	@objcopy --redefine-syms=$(REFDIR)/obj/pecan/$*_syms.txt $< $@
$(REFDIR)/obj/cactus_pecan_harvest.o: $(HERE)../shim/cactus_pecan_harvest.c
	@mkdir -p $(REFDIR)/obj
	@$(CC) -c $(FL_CFLAGS) -Wall -Wno-unused-function $< -o $@

FL_PECAN_HARVEST_OBJS := $(REFDIR)/obj/flower_harness.o $(FL_COMMON) $(REFDIR)/obj/poaBarAligner.o \
                         $(REFDIR)/obj/pecan/pairwiseAligner_hweak.o $(REFDIR)/obj/pecan/pairwiseAligner_private.o \
                         $(REFDIR)/obj/pecan/multipleAligner_hweak.o $(REFDIR)/obj/pecan/multipleAligner_private.o \
                         $(REFDIR)/obj/cactus_pecan_harvest.o
$(REFDIR)/libflower_pecan_harvest.so: $(FL_PECAN_HARVEST_OBJS) $(HERE)gen_stubs_all.sh
	@sh $(HERE)gen_stubs_all.sh $(FL_PECAN_HARVEST_OBJS) > $(REFDIR)/obj/flower_pecan_harvest_stubs.c
	@$(CC) -shared $(FL_CFLAGS) -o $@ $(FL_PECAN_HARVEST_OBJS) $(REFDIR)/obj/flower_pecan_harvest_stubs.c -lm -lz -lpthread
