# Oracle build recipe of the map merge (TEST INFRASTRUCTURE), run after oracle/Makefile by __graft_entry__.build():
#
#   _ref/libmerge_b200.so   the reference's Karto / Mapper objects and oracle/ref_driver.cpp (built by oracle/Makefile),
#                           oracle/merge_ref_driver.cpp (the tool's transformScan restated with Karto's setters) and
#                           integration/merge_maps_driver.cpp (the map-merge binding, integration/merge_maps_b200.hpp);
#                           links ../slam_toolbox_b200/lib/libb200slam.so.  Only when the reference sources are present.
#
#     make -C oracle -f merge.mk
REF ?= $(abspath ../../reference)
CXX := g++
OUT := _ref
INTEG := ../integration
CXXFLAGS := -std=c++17 -O2 -fPIC -w -ffp-contract=off -pthread
LIBDIR := $(abspath ../slam_toolbox_b200/lib)
LDLIBS := -L$(LIBDIR) -lb200slam -Wl,-rpath,'$$ORIGIN/../../slam_toolbox_b200/lib'
INC := -Istubs -I$(REF)/lib/karto_sdk/include -I../include

ifneq ($(wildcard $(REF)/lib/karto_sdk/src/Mapper.cpp),)
all: $(OUT)/libmerge_b200.so
$(OUT)/merge_ref_driver.o: merge_ref_driver.cpp
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INC) -c $< -o $@
$(OUT)/merge_maps_driver.o: $(INTEG)/merge_maps_driver.cpp $(INTEG)/merge_maps_b200.hpp $(INTEG)/occupancy_b200.hpp \
                            ../include/b200slam.h
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INC) -c $< -o $@
$(OUT)/libmerge_b200.so: $(OUT)/merge_maps_driver.o $(OUT)/merge_ref_driver.o $(OUT)/ref_driver.o $(OUT)/Karto.o $(OUT)/Mapper.o \
                         $(LIBDIR)/libb200slam.so
	$(CXX) -shared -pthread -o $@ $(OUT)/merge_maps_driver.o $(OUT)/merge_ref_driver.o $(OUT)/ref_driver.o $(OUT)/Karto.o \
	  $(OUT)/Mapper.o $(LDLIBS)
else
all:
	@echo "oracle/merge.mk: $(REF) not present; keeping the map-merge library already in $(OUT)/ (if any)"
endif

.PHONY: all
