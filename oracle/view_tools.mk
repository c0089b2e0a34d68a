# Builds the reference's python/depthmotionnet/dataset_tools/view_tools_cython.pyx (test infrastructure): cythonized
# unmodified from where it lies (the reference tree that REF_SRC, its lmbspecialops/src, belongs to) into _ref/ and
# compiled as the Python extension _ref/view_tools_cython.so.  Nothing is copied into this repository.
#   make -C oracle -f view_tools.mk REF_SRC=<reference>/lmbspecialops/src
CC ?= gcc
PYTHON ?= python3
REF_SRC ?= $(DEMON_REF_SRC)
VIEW_TOOLS_PYX ?= $(REF_SRC)/../../python/depthmotionnet/dataset_tools/view_tools_cython.pyx
PY_INC ?= $(shell $(PYTHON) -c "import sysconfig; print(sysconfig.get_paths()['include'])")
NP_INC ?= $(shell $(PYTHON) -c "import numpy; print(numpy.get_include())")

view_tools: _ref/view_tools_cython.so

_ref/view_tools_cython.so: $(VIEW_TOOLS_PYX) view_tools.mk
	mkdir -p _ref
	$(PYTHON) -m cython -3 -o _ref/view_tools_cython.c $(VIEW_TOOLS_PYX)
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -w -I $(PY_INC) -I $(NP_INC) -o $@ _ref/view_tools_cython.c

.PHONY: view_tools
