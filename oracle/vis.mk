# Builds the reference's python/depthmotionnet/vis_cython.pyx (test infrastructure): cythonized unmodified from where it
# lies (the reference tree that REF_SRC, its lmbspecialops/src, belongs to) into _ref/ and compiled as the Python
# extension _ref/vis_cython.so.  Nothing is copied into this repository.
#   make -C oracle -f vis.mk REF_SRC=<reference>/lmbspecialops/src
CC ?= gcc
PYTHON ?= python3
REF_SRC ?= $(DEMON_REF_SRC)
VIS_PYX ?= $(REF_SRC)/../../python/depthmotionnet/vis_cython.pyx
PY_INC ?= $(shell $(PYTHON) -c "import sysconfig; print(sysconfig.get_paths()['include'])")
NP_INC ?= $(shell $(PYTHON) -c "import numpy; print(numpy.get_include())")

vis: _ref/vis_cython.so

_ref/vis_cython.so: $(VIS_PYX) vis.mk
	mkdir -p _ref
	$(PYTHON) -m cython -3 -o _ref/vis_cython.c $(VIS_PYX)
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -w -I $(PY_INC) -I $(NP_INC) -o $@ _ref/vis_cython.c

.PHONY: vis
