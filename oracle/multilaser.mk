# Oracle build recipe of the multi-laser occupancy grid (TEST INFRASTRUCTURE), run after oracle/Makefile by
# __graft_entry__.build():
#
#   _ref/libmultilaser_ref.so   the reference's Karto / Mapper objects, oracle/ref_driver.cpp, oracle/merge_ref_driver.cpp and
#                               integration/merge_maps_driver.cpp (the map-merge binding; all built by oracle/Makefile and
#                               oracle/merge.mk) and oracle/multilaser_ref_driver.cpp (named lasers, scans on a chosen laser);
#                               links ../slam_toolbox_b200/lib/libb200slam.so.  Only when the reference sources are present.
#
#     make -C oracle -f multilaser.mk
REF ?= $(abspath ../../reference)
CXX := g++
OUT := _ref
CXXFLAGS := -std=c++17 -O2 -fPIC -w -ffp-contract=off -pthread
INC := -Istubs -I$(REF)/lib/karto_sdk/include
LIBDIR := $(abspath ../slam_toolbox_b200/lib)
LDLIBS := -L$(LIBDIR) -lb200slam -Wl,-rpath,'$$ORIGIN/../../slam_toolbox_b200/lib'

ifneq ($(wildcard $(REF)/lib/karto_sdk/src/Mapper.cpp),)
all: $(OUT)/libmultilaser_ref.so
$(OUT)/multilaser_ref_driver.o: multilaser_ref_driver.cpp
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INC) -c $< -o $@
ML_OBJS := $(OUT)/multilaser_ref_driver.o $(OUT)/merge_maps_driver.o $(OUT)/merge_ref_driver.o $(OUT)/ref_driver.o $(OUT)/Karto.o \
           $(OUT)/Mapper.o
$(OUT)/libmultilaser_ref.so: $(ML_OBJS) $(LIBDIR)/libb200slam.so
	$(CXX) -shared -pthread -o $@ $(ML_OBJS) $(LDLIBS)
else
all:
	@echo "oracle/multilaser.mk: $(REF) not present; keeping the multi-laser library already in $(OUT)/ (if any)"
endif

.PHONY: all
