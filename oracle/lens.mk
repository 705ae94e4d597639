# oracle/lens.mk -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -C oracle -f lens.mk  -> oracle/_ref/libref_lens_strict.so, oracle/_ref/libref_lens_fast.so
#
# The reference's own lines for lens correction (ref_shim/lens/ref_lens.c), cut verbatim by slice.py and compiled in place from $(REF)
# with the strict and the release flags of oracle/Makefile, beside src/external/LensSerious/src/lensserious.c, unmodified:
#     iop/lens.c :121-167 the correction enums, :392-409 dt_iop_lensfun_data_t, :620-653 get_modifier, :680-923 process()
#     pixel/interpolation.h :37-67 the interpolator types
#     pixel/interpolation.c :51-70 border modes, :88-165 _clip and _prepare_tap_boundaries, :175-287 the three tap generators,
#                           :298-314 their table, :320-342 _compute_upsampling_kernel, :393-489 dt_interpolation_compute_sample,
#                           :600-665 dt_interpolation_new
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := lens
LENS_SO := $(HERE)_ref/libref_lens_strict.so
LS := $(REF)/src/external/LensSerious

.PHONY: lens
lens:
	@if [ -d "$(REF)/src" ] && [ -f $(LENS_SO) ] && [ -z "$$(find $(HERE)ref_shim/lens $(HERE)lens.mk -newer $(LENS_SO) -print -quit)" ]; then \
	  echo "oracle/_ref/libref_lens_*.so are up to date"; \
	elif [ -d "$(REF)/src" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(SLICE) $(REF)/src/pixel/interpolation.h $(HERE)_ref/gen_lens_interpolation.c 37-67 && \
	  $(SLICE) $(REF)/src/pixel/interpolation.c $(HERE)_ref/gen_lens_itor.c 51-70 88-165 175-287 298-314 320-342 393-489 600-665 && \
	  cat $(HERE)_ref/gen_lens_itor.c >> $(HERE)_ref/gen_lens_interpolation.c && rm $(HERE)_ref/gen_lens_itor.c && \
	  $(SLICE) $(REF)/src/iop/lens.c $(HERE)_ref/gen_lens.c 121-167 392-409 620-653 680-923 && \
	  $(HOSTCC) $(REF_FAST) $(REF_INC) -I$(LS)/include -w -shared -fPIC -o $(HERE)_ref/libref_lens_fast.so $(HERE)ref_shim/lens/ref_lens.c $(LS)/src/lensserious.c -lm && \
	  $(HOSTCC) $(REF_STRICT) $(REF_INC) -I$(LS)/include -w -shared -fPIC -o $(LENS_SO) $(HERE)ref_shim/lens/ref_lens.c $(LS)/src/lensserious.c -lm && \
	  rm -f $(HERE)_ref/gen_lens*.c && \
	  echo "built oracle/_ref/libref_lens_*.so from $(REF)"; \
	else echo "no $(REF): keeping prebuilt oracle/_ref/libref_lens_*.so (if any)"; fi
