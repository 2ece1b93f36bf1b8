# The reference's TournamentResult (engine/src/rl/tournamentresult.{h,cpp}), compiled unchanged from its own sources
# behind the C entry point of ref/tournament_shim.cpp.  Like the `ref` target of the Makefile beside this one: built
# from where the sources lie under $(REFERENCE), output to _ref/ only (git-ignored); nothing of the reference is copied
# into this repository.  tests/test_match_host_logic.py pins crazyara_b200/match.py::TournamentResult with it.
#     make -C oracle -f ref_tournament.mk
REFERENCE ?= /root/reference
REF_SRC := $(REFERENCE)/engine/src
_ref/libref_tournament.so: ref/tournament_shim.cpp $(REF_SRC)/rl/tournamentresult.cpp
	@mkdir -p _ref
	g++ -O2 -fPIC -std=c++17 -w -I$(REF_SRC) -shared -o $@ $^
