// Stand-in for iod/symbols.hh (included by vpp/algorithms/distance_transforms/distance_transforms.hh): the symbols live in the
// iod/symbol.hh stand-in of this directory.
#pragma once
#include <iod/symbol.hh>
