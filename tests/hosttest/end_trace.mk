# TEST-ONLY: the CPU stand-in for libbarb200 (standin_device.cpp) with a trace layer (standin_trace.cpp), under the product's real
# host_bar.cpp and host_end_trace.cpp: the no-GPU suite runs barb200_trace_ends' window rounds on it
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CSRC := $(HERE)../../cactus_b200/csrc
.PHONY: end_trace
end_trace: $(HERE)_build/libbarb200_trace_standin.so
$(HERE)_build/libbarb200_trace_standin.so: $(HERE)standin_trace.cpp $(HERE)standin_device.cpp $(HERE)hosttest.cpp $(CSRC)/host_bar.cpp $(CSRC)/host_end_trace.cpp $(CSRC)/poa_graph.cuh $(CSRC)/poa_types.h $(CSRC)/guide_tree.cuh $(CSRC)/slot_plan.h $(CSRC)/stage_plan.h $(CSRC)/poa_kernel.cuh $(CSRC)/end_queue.h $(CSRC)/bar_windows.h $(CSRC)/host_api.h $(CSRC)/pecan_plan.cpp $(HERE)../../include/barb200.h
	@mkdir -p $(HERE)_build
	g++ -O2 -std=c++17 -fPIC -shared -Wall -ffp-contract=off -pthread -fopenmp -x c++ -o $@ $(HERE)standin_trace.cpp $(HERE)hosttest.cpp $(CSRC)/host_bar.cpp $(CSRC)/host_end_trace.cpp $(CSRC)/pecan_plan.cpp
