# oracle/colorbalancergb.mk -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -C oracle -f colorbalancergb.mk  -> oracle/_ref/libref_colorbalancergb_strict.so, oracle/_ref/libref_colorbalancergb_fast.so
#
# The reference's own lines for colour balance rgb (ref_shim/colorbalancergb/ref_colorbalancergb.c), cut verbatim by slice.py and
# compiled in place from $(REF) with the strict and the release flags of oracle/Makefile:
#     iop/colorbalancergb.c :70-78 LUT_ELEM, STEPS, DEG_TO_RAD; :82-192 the enums, params, GUI and data structs; :509-927 opacity_masks, soft_clip,
#                           lookup_gamut, process(); :1096-1353 Delta_H, commit_params()
# over common/colorspaces_inline_conversions.h, math/matrices.h, system/simd.h, math/math.h and pixel/chromatic_adaptation.h, unmodified.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := colorbalancergb
CBRGB_SO := $(HERE)_ref/libref_colorbalancergb_strict.so

.PHONY: colorbalancergb
colorbalancergb:
	@if [ -d "$(REF)/src" ] && [ -f $(CBRGB_SO) ] && [ -z "$$(find $(HERE)ref_shim/colorbalancergb $(HERE)colorbalancergb.mk -newer $(CBRGB_SO) -print -quit)" ]; then \
	  echo "oracle/_ref/libref_colorbalancergb_*.so are up to date"; \
	elif [ -d "$(REF)/src" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(SLICE) $(REF)/src/iop/colorbalancergb.c $(HERE)_ref/gen_colorbalancergb.c 70-78 82-192 509-927 1096-1353 && \
	  $(HOSTCC) $(REF_FAST) $(REF_INC) -w -shared -fPIC -o $(HERE)_ref/libref_colorbalancergb_fast.so $(HERE)ref_shim/colorbalancergb/ref_colorbalancergb.c -lm && \
	  $(HOSTCC) $(REF_STRICT) $(REF_INC) -w -shared -fPIC -o $(CBRGB_SO) $(HERE)ref_shim/colorbalancergb/ref_colorbalancergb.c -lm && \
	  rm -f $(HERE)_ref/gen_colorbalancergb.c && \
	  echo "built oracle/_ref/libref_colorbalancergb_*.so from $(REF)"; \
	else echo "no $(REF): keeping prebuilt oracle/_ref/libref_colorbalancergb_*.so (if any)"; fi
