# oracle/event.mk - TEST INFRASTRUCTURE ONLY.
#
# Builds, into oracle/_ref/ (git-ignored; travels with the working tree to a GPU machine):
#   test_event       the reference's own event-queue test program (test/test_event.c with its test/test.h), compiled UNMODIFIED
#                    from where it lies and linked against _ref/libcimba_ref.so: `test_event -s <seed>` prints the text of
#                    test/reference/event.txt for that seed;
#   libeventdrv.so   ref_build/event_driver.c: test_events()'s sequence against the unmodified reference library, returning the
#                    counters and pop trace of examples/event_model.cuh's EventTestT.
# Run after `make -C oracle all`:
#
#     make -C oracle -f event.mk
#
# Like oracle/Makefile it builds nothing where the reference sources are absent.  Same flags as oracle/Makefile's librefdrv.so.
REF     ?= /root/reference
OUT     := _ref
CC      := gcc
STD     := -std=c2x -Wno-pedantic -D_POSIX_C_SOURCE=200809L -D_GNU_SOURCE
RELDEFS := -DNMXCSR -DNDEBUG -DNLOGINFO -DNASSERT
INC     := -I$(REF)/include -I$(REF)/src -I$(OUT)/gen

.PHONY: all
all: $(if $(wildcard $(REF)/src/cimba.c),$(OUT)/test_event $(OUT)/libeventdrv.so,)

$(OUT)/test_event: $(REF)/test/test_event.c $(REF)/test/test.h $(OUT)/libcimba_ref.so
	$(CC) $(STD) $(RELDEFS) -O2 $(INC) -I$(REF)/test $(REF)/test/test_event.c \
	    -o $@ -L$(OUT) -lcimba_ref -Wl,-rpath,'$$ORIGIN' -lm -lpthread

$(OUT)/libeventdrv.so: ref_build/event_driver.c $(OUT)/libcimba_ref.so
	$(CC) $(STD) $(RELDEFS) -O3 -fPIC -shared $(INC) ref_build/event_driver.c \
	    -o $@ -L$(OUT) -lcimba_ref -Wl,-rpath,'$$ORIGIN' -lm -lpthread
