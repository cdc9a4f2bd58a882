# The SDF-program harness over the reference (tests/harness/vxh_programs.cpp + vxh_capi.cpp, linked with the UNMODIFIED
# reference objects of `make -C oracle ref`):
#
#   make -C oracle -f programs.mk programs   -> _ref/libvxh_programs_ref.so
#
# One library holds the reference's grids and both sources' calls (tests/program_harness.py), so a grid made with a program
# is read back, edited and polygonized by the same copy of the reference.  Variables and the reference objects come from
# the Makefile of this directory.
include Makefile

PROGRAMS := $(OUT)/libvxh_programs_ref.so

programs: $(PROGRAMS)

$(PROGRAMS): ../tests/harness/vxh_programs.cpp ../tests/harness/vxh_capi.cpp ../voxels_b200/csrc/vxb_program.h \
             ../voxels_b200/csrc/vxb_surfaces.h ../include/vxb200.h $(OBJS)
	$(CXX) $(CXXFLAGS) -DVXH_WITH_INTERNAL_GRID -I $(REF)/src -shared -o $@ ../tests/harness/vxh_capi.cpp ../tests/harness/vxh_programs.cpp $(OBJS)

.PHONY: programs
