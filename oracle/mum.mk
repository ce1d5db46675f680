# oracle/mum.mk -- the CHECKERS of K5 (MUM anchors, cactus_b200/csrc/mum_anchor.cu), on top of oracle/Makefile's variables and
# reference objects (run after it: make -C oracle -f mum.mk):
#
#   _build/libmum_oracle.so        plain-C restatement of cPecan's MUM anchoring (mum_oracle.c); always buildable.
#   _ref/libmum_ref.so             the UNMODIFIED reference pairwiseAligner.o (+ stateMachine.o, multipleAligner.o, sonLib)
#                                  behind mum_ref_harness.c. Only built where the reference sources exist.
#   _ref/libflower_standin_mum.so  the flower-level drop-in build of oracle/Makefile (FL_SHIM_OBJS: the real shims under the
#                                  reference's flower code) over tests/hosttest's stand-in device WITH the host build of K5
#                                  (tests/hosttest/mum.mk: libbarb200_standin_mum.so), so that the no-GPU suite runs cPecan
#                                  bar() on adjacencies long enough for MUM anchoring.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := mum
.PHONY: mum mum_ref

mum: $(BLDDIR)/libmum_oracle.so mum_ref

$(BLDDIR)/libmum_oracle.so: $(HERE)mum_oracle.c
	@mkdir -p $(BLDDIR)
	@$(CC) -O2 -fPIC -shared -std=gnu99 -Wall -o $@ $<

STANDIN_MUM_LIB := $(HERE)../tests/hosttest/_build/libbarb200_standin_mum.so
ifneq ($(wildcard $(ABPOA)/src/abpoa_align.c),)
mum_ref: $(REFDIR)/libmum_ref.so $(REFDIR)/libflower_standin_mum.so
else
mum_ref:
	@echo "oracle/mum.mk: $(REFERENCE) not present; keeping prebuilt oracle/_ref (if any)"
endif

$(REFDIR)/libmum_ref.so: $(REFDIR)/obj/pecan/pairwiseAligner.o $(PECAN_OBJS) $(SONLIB_OBJS) $(HERE)mum_ref_harness.c
	@$(CC) -O2 -fPIC -shared -fopenmp -std=gnu99 -w -UNDEBUG $(PECAN_INC) -o $@ $(HERE)mum_ref_harness.c \
	    $(REFDIR)/obj/pecan/pairwiseAligner.o $(PECAN_OBJS) $(SONLIB_OBJS) -lm -lz -lpthread

ifneq ($(wildcard $(STANDIN_MUM_LIB)),)
$(REFDIR)/libflower_standin_mum.so: $(FL_SHIM_OBJS) $(STANDIN_MUM_LIB) $(HERE)gen_stubs_all.sh
	@sh $(HERE)gen_stubs_all.sh $(FL_SHIM_OBJS) -L$(HERE)../tests/hosttest/_build -lbarb200_standin_mum > $(REFDIR)/obj/flower_standin_mum_stubs.c
	@$(CC) -shared $(FL_CFLAGS) -o $@ $(FL_SHIM_OBJS) $(REFDIR)/obj/flower_standin_mum_stubs.c \
	    -L$(HERE)../tests/hosttest/_build -lbarb200_standin_mum -Wl,-rpath,'$$ORIGIN/../../tests/hosttest/_build' -lm -lz -lpthread
else
$(REFDIR)/libflower_standin_mum.so:
	@echo "oracle/mum.mk: tests/hosttest/mum.mk's stand-in not built yet; skipping libflower_standin_mum.so"
endif
