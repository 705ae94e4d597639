# oracle/fdc.mk -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -C oracle -f fdc.mk  -> oracle/_ref/libref_fdc_strict.so, oracle/_ref/libref_fdc_fast.so
#
# The reference's own lines for frequency-domain chroma on X-Trans sensors (ref_shim/fdc/ref_fdc.c), cut verbatim by slice.py and
# compiled in place from $(REF) with the strict and the release flags of oracle/Makefile:
#     iop/demosaic/markesteijn.c :25-26 SQR, :29-40 hexmap, :525-1639 xtrans_fdc_interpolate; :548-1071 its coefficient tables once more,
#                                on their own, so that the wrapper can hand them out
#     develop/imageop_math.h :175-219 FC, FCxtrans
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile
.DEFAULT_GOAL := fdc
FDC_SO := $(HERE)_ref/libref_fdc_strict.so

.PHONY: fdc
fdc:
	@if [ -d "$(REF)/src" ] && [ -f $(FDC_SO) ] && [ -z "$$(find $(HERE)ref_shim/fdc $(HERE)fdc.mk -newer $(FDC_SO) -print -quit)" ]; then \
	  echo "oracle/_ref/libref_fdc_*.so are up to date"; \
	elif [ -d "$(REF)/src" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(SLICE) $(REF)/src/develop/imageop_math.h $(HERE)_ref/gen_fdc_imageop_math.c 175-219 && \
	  $(SLICE) $(REF)/src/iop/demosaic/markesteijn.c $(HERE)_ref/gen_fdc.c 25-26 29-40 525-1639 && \
	  $(SLICE) $(REF)/src/iop/demosaic/markesteijn.c $(HERE)_ref/gen_fdc_tables.c 548-1071 && \
	  $(HOSTCC) $(REF_FAST) $(REF_INC) -w -shared -fPIC -o $(HERE)_ref/libref_fdc_fast.so $(HERE)ref_shim/fdc/ref_fdc.c -lm && \
	  $(HOSTCC) $(REF_STRICT) $(REF_INC) -w -shared -fPIC -o $(FDC_SO) $(HERE)ref_shim/fdc/ref_fdc.c -lm && \
	  rm -f $(HERE)_ref/gen_fdc*.c && \
	  echo "built oracle/_ref/libref_fdc_*.so from $(REF)"; \
	else echo "no $(REF): keeping prebuilt oracle/_ref/libref_fdc_*.so (if any)"; fi
