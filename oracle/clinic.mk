# oracle/clinic.mk - TEST INFRASTRUCTURE ONLY.
#
# Builds oracle/_ref/libclinicdrv.so (git-ignored; travels with the working tree to a GPU machine): the walk-in clinic of
# examples/clinic_model.cuh written against the UNMODIFIED reference library (ref_build/clinic_driver.c), linked against
# the _ref/libcimba_ref.so that oracle/Makefile builds.  Run after `make -C oracle all`:
#
#     make -C oracle -f clinic.mk
#
# Like oracle/Makefile it builds nothing where the reference sources are absent.  Same flags as oracle/Makefile's
# librefdrv.so.
REF     ?= /root/reference
OUT     := _ref
CC      := gcc
STD     := -std=c2x -Wno-pedantic -D_POSIX_C_SOURCE=200809L -D_GNU_SOURCE
RELDEFS := -DNMXCSR -DNDEBUG -DNLOGINFO -DNASSERT
INC     := -I$(REF)/include -I$(REF)/src -I$(OUT)/gen

.PHONY: all
all: $(if $(wildcard $(REF)/src/cimba.c),$(OUT)/libclinicdrv.so,)

$(OUT)/libclinicdrv.so: ref_build/clinic_driver.c $(OUT)/libcimba_ref.so
	$(CC) $(STD) $(RELDEFS) -O3 -fPIC -shared $(INC) ref_build/clinic_driver.c \
	    -o $@ -L$(OUT) -lcimba_ref -Wl,-rpath,'$$ORIGIN' -lm -lpthread
