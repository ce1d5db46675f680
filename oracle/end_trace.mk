# oracle/end_trace.mk -- the CHECKERS of barb200_trace_ends (every window of every end), on top of oracle/Makefile's variables and
# reference objects (run after it: make -C oracle -f end_trace.mk):
#
#   _build/libend_trace_oracle.so  oracle_trace_ends: bar_oracle.c's restated window chain and cross-end trim with every window's
#                                  job run through poa_oracle.c's traced MSA (end_trace_oracle.c); always buildable.
#   _ref/libbar_trace_ref.so       the UNMODIFIED reference poaBarAligner.o linked with -Wl,--wrap=abpoa_msa (and the allocation
#                                  and window-list calls of its loop) behind end_trace_ref_harness.c: the window inputs, job
#                                  traces and trims of the reference's own loop. Only built where the reference sources exist.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := end_trace
.PHONY: end_trace end_trace_ref

end_trace: $(BLDDIR)/libend_trace_oracle.so end_trace_ref

$(BLDDIR)/libend_trace_oracle.so: $(HERE)end_trace_oracle.c $(HERE)bar_oracle.c $(HERE)poa_oracle.c $(HERE)poa_oracle.h
	@mkdir -p $(BLDDIR)
	@$(CC) -O2 -fPIC -shared -std=gnu99 -Wall -fopenmp -ffp-contract=off -o $@ $(HERE)poa_oracle.c $(HERE)end_trace_oracle.c -lm

ifneq ($(wildcard $(ABPOA)/src/abpoa_align.c),)
end_trace_ref: $(REFDIR)/libbar_trace_ref.so
else
end_trace_ref:
	@echo "oracle/end_trace.mk: $(REFERENCE) not present; keeping prebuilt oracle/_ref (if any)"
endif

$(REFDIR)/obj/ref_harness_trace.o: $(HERE)ref_harness.c
	@mkdir -p $(REFDIR)/obj
	@$(CC) -c -O2 -fPIC -fopenmp $(ABPOA_FLAGS) -w $< -o $@
$(REFDIR)/obj/end_trace_ref_harness.o: $(HERE)end_trace_ref_harness.c $(HERE)bar_ref_harness.c
	@mkdir -p $(REFDIR)/obj
	@$(CC) -c -O2 -fPIC -fopenmp -std=gnu99 -Wall -Wno-unused-function -UNDEBUG $(BAR_INC) $< -o $@

# stubs.c: the abort() stubs of libbar_ref.so for the Flower-level Cactus API poaBarAligner.o references and never calls here
$(REFDIR)/libbar_trace_ref.so: $(REFDIR)/obj/end_trace_ref_harness.o $(REFDIR)/obj/ref_harness_trace.o $(REFDIR)/obj/poaBarAligner.o \
                               $(SONLIB_OBJS) $(ABPOA_OBJS) $(REFDIR)/libbar_ref.so
	@$(CC) -O2 -fPIC -shared -fopenmp -std=gnu99 -w -o $@ $(REFDIR)/obj/end_trace_ref_harness.o $(REFDIR)/obj/ref_harness_trace.o \
	    $(REFDIR)/obj/stubs.c $(REFDIR)/obj/poaBarAligner.o $(SONLIB_OBJS) $(ABPOA_OBJS) \
	    -Wl,--wrap=abpoa_msa,--wrap=st_calloc,--wrap=stList_append,--wrap=stList_destruct -lm -lz -lpthread
