# oracle/ref_volume.mk -- TEST INFRASTRUCTURE ONLY: builds oracle/ref_volume_map.cpp against the reference's own, unmodified library sources
# and GenerateDensityMap's quadrature into oracle/_ref/bin/RefGenerateVolumeMap, only when the reference sources are present; outputs only
# under oracle/_ref/ (git-ignored).  The reference build recipe (REF, CXX, REFINC, REFLIBSRC, REFFLAGS) is oracle/Makefile's own, included
# here rather than restated, so the two cannot drift apart.  The generator needs none of oracle/Makefile's generated files, so running
# this next to `make -C oracle all` writes nothing the other writes.
#   make -C oracle -f ref_volume.mk
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

QUAD := $(REF)/cmd/generate_density_map/gauss_quadrature.cpp

ifneq ($(wildcard $(QUAD)),)
ref_volume_map: $(HERE)_ref/bin/RefGenerateVolumeMap
$(HERE)_ref/bin/RefGenerateVolumeMap: $(HERE)ref_volume_map.cpp $(QUAD) $(REFLIBSRC) $(HERE)ref_eigen/Eigen/Dense
	mkdir -p $(HERE)_ref/bin
	$(CXX) $(REFFLAGS) $(REFINC) -I$(REF)/cmd/generate_density_map -o $@ $(HERE)ref_volume_map.cpp $(QUAD) $(REFLIBSRC)
else
ref_volume_map:
	@echo "reference not present at $(REF): keeping prebuilt oracle/_ref (if any)"
endif
.DEFAULT_GOAL := ref_volume_map
.PHONY: ref_volume_map
