# oracle/scaled.mk -- TEST INFRASTRUCTURE ONLY: the checkers of the reduced-size (1/2, 1/4, 1/8) JPEG decoder.
#
#  _ref/libjpeg_scaled_oracle.so : jpeg_scaled_oracle.c, the C restatement of libjpeg-turbo's scaled decoding, on
#                                  top of jpeg_oracle.c (entropy decoder, islow IDCT).  Always buildable.
#  _ref/libjpeg_scaled_ref.so    : jpeg_scaled_ref.c, a harness over the real libjpeg-turbo binary that Makefile's
#                                  _ref/libuhdr_ref_turbo.so links (Pillow's, copied next to it and found through an
#                                  $ORIGIN rpath, so the pair travels with _ref/).  Built only where that binary is.
# Outputs only under _ref/ (git-ignored).  Run by __graft_entry__.build() after Makefile.
CC = gcc
ORACLE_CFLAGS = -O2 -m64 -march=x86-64 -mtune=generic -ffp-contract=off -fPIC -Wall -Wextra
TURBO_LIB ?= $(firstword $(wildcard $(shell python3 -c "import PIL,os;print(os.path.join(os.path.dirname(os.path.dirname(PIL.__file__)),'pillow.libs'))" 2>/dev/null)/libjpeg-*.so.62*))

all: _ref/libjpeg_scaled_oracle.so harness

_ref/libjpeg_scaled_oracle.so: jpeg_scaled_oracle.c jpeg_oracle.c jpeg_oracle.h
	@mkdir -p _ref
	$(CC) $(ORACLE_CFLAGS) -std=c11 -shared -o $@ jpeg_scaled_oracle.c jpeg_oracle.c -lm

harness:
	@if [ -n "$(TURBO_LIB)" ]; then $(MAKE) --no-print-directory -f scaled.mk _ref/libjpeg_scaled_ref.so; \
	 else echo "oracle: no libjpeg-turbo binary found (Pillow's pillow.libs), skipping _ref/libjpeg_scaled_ref.so"; fi

_ref/libjpeg_scaled_ref.so: jpeg_scaled_ref.c ref_turbo/jpeglib.h
	@mkdir -p _ref
	@cp -f $(TURBO_LIB) _ref/$(notdir $(TURBO_LIB))
	$(CC) $(ORACLE_CFLAGS) -std=c11 -Iref_turbo -shared -Wl,-rpath,'$$ORIGIN' -o $@ jpeg_scaled_ref.c _ref/$(notdir $(TURBO_LIB))

.PHONY: all harness
