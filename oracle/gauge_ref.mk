# TEST INFRASTRUCTURE ONLY.
#   make -f gauge_ref.mk : oracle/_ref/libquda_gaugeref.so -- the reference's host gauge force
#                          (tests/host_reference/gauge_force_reference.cpp) and mom_action (tests/utils/host_utils.cpp),
#                          compiled in place with the flags and the link-time stand-ins of libquda_hostref.so (Makefile,
#                          ref_glue.cpp) and exported through gauge_glue.cpp.  A library of its own, so that the pinned
#                          Dslash oracle keeps exactly the link set it was pinned with.
include Makefile

GAUGESRC = $(REF)/tests/host_reference/gauge_force_reference.cpp
GAUGEOBJ = $(REFOBJ) $(R)/obj/gauge_force_reference.o $(R)/obj/ref_glue.o $(R)/obj/gauge_glue.o

gaugeref: $(R)/libquda_gaugeref.so

$(R)/obj/gauge_glue.o: gauge_glue.cpp $(R)/gen/quda_define.h
	$(REFCXX) -fvisibility=hidden -c gauge_glue.cpp -o $@

$(R)/libquda_gaugeref.so: $(GAUGEOBJ) ref_exports.map
	$(CXX) -shared $(OMP) -o $@ $(GAUGEOBJ) \
	  -Wl,--gc-sections -Wl,--version-script=ref_exports.map -Wl,--no-undefined -lm

.DEFAULT_GOAL := gaugeref
.PHONY: gaugeref
