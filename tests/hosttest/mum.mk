# TEST-ONLY host builds of K5 (cactus_b200/csrc/mum_anchor.cuh + mum_plan.h, driven by mum_host.cpp), run after the Makefile here
# (make -C tests/hosttest -f mum.mk):
#   _build/libmum_host.so               the host build alone (tests/_mumlib.py)
#   _build/libbarb200_standin_mum.so    the stand-in device of the Makefile here (standin_device.cpp) plus the MUM anchor entries
#                                       (standin_mum.cpp), for oracle/mum.mk's flower-level build
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CSRC := $(HERE)../../cactus_b200/csrc
.PHONY: mum
mum: $(HERE)_build/libmum_host.so $(HERE)_build/libbarb200_standin_mum.so
MUM_DEPS := $(HERE)mum_host.cpp $(CSRC)/mum_anchor.cuh $(CSRC)/mum_plan.h
$(HERE)_build/libmum_host.so: $(MUM_DEPS)
	@mkdir -p $(HERE)_build
	g++ -O2 -std=c++17 -fPIC -shared -Wall -o $@ $(HERE)mum_host.cpp
$(HERE)_build/libbarb200_standin_mum.so: $(MUM_DEPS) $(HERE)standin_mum.cpp $(HERE)standin_device.cpp $(HERE)hosttest.cpp $(CSRC)/poa_graph.cuh $(CSRC)/poa_types.h $(CSRC)/guide_tree.cuh $(CSRC)/slot_plan.h $(CSRC)/stage_plan.h $(CSRC)/poa_kernel.cuh $(CSRC)/host_bar.cpp $(CSRC)/end_queue.h $(CSRC)/bar_windows.h $(CSRC)/host_api.h $(CSRC)/pecan_plan.cpp $(HERE)../../include/barb200.h
	@mkdir -p $(HERE)_build
	g++ -O2 -std=c++17 -fPIC -shared -Wall -ffp-contract=off -pthread -fopenmp -x c++ -o $@ $(HERE)standin_device.cpp $(HERE)hosttest.cpp $(CSRC)/host_bar.cpp $(CSRC)/pecan_plan.cpp $(HERE)mum_host.cpp $(HERE)standin_mum.cpp
