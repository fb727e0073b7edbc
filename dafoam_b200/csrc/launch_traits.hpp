// Resident CTAs per SM (the second __launch_bounds__ argument, which caps the registers per thread) of the cell-per-thread
// kernels.  Kept apart from solver.hpp so that a translation unit can instantiate one kernel with the product's launch bounds
// and read its register use (`nvcc -Xptxas -v`) in seconds (tests/test_kernel_resources.py).
#pragma once
#include "backend.hpp"
#include "fwd_kernels.hpp"
#include "rev_kernels.hpp"
#include "comp_kernels.hpp"
#include "comp_rev_kernels.hpp"
#include "primal_kernels.hpp"
#include "comp_primal_kernels.hpp"

namespace dab
{

#if !defined(DAB_HOSTSIM)
// RevB: at 2 CTAs per SM (up to 255 registers) a face's whole load block stays in registers; at 3 (168 registers) the kernel
// spills and is 40 % slower on the H100, at 4 (128) more than twice as slow (DESIGN.md section 4)
#ifndef DAB_REVB_MINBLOCKS
#define DAB_REVB_MINBLOCKS 2
#endif
#ifndef DAB_FWDB_MINBLOCKS
#define DAB_FWDB_MINBLOCKS 3
#endif
template <int NF, int FEAT> struct LaunchTraits<RevB<NF, FEAT>> { static constexpr int minBlocks = DAB_REVB_MINBLOCKS; };
// with the hoisted load blocks: RevA 96 registers / 5 CTAs per SM, RevC 128 / 4
template <int NF> struct LaunchTraits<RevA<NF>> { static constexpr int minBlocks = 5; };
template <int NF> struct LaunchTraits<RevC<NF>> { static constexpr int minBlocks = 4; };
template <int NF, int FEAT> struct LaunchTraits<FwdB<NF, FEAT>> { static constexpr int minBlocks = DAB_FWDB_MINBLOCKS; };
template <int NF, int FEAT> struct LaunchTraits<UEqnAssemble<NF, FEAT>> { static constexpr int minBlocks = DAB_FWDB_MINBLOCKS; };
template <int NF> struct LaunchTraits<NutEqnAssemble<NF>> { static constexpr int minBlocks = 4; };
template <int NF> struct LaunchTraits<cFwdB<NF>> { static constexpr int minBlocks = 2; };
template <int NF> struct LaunchTraits<cUEqnAssemble<NF>> { static constexpr int minBlocks = 2; };
template <int NF> struct LaunchTraits<cEEqnAssemble<NF>> { static constexpr int minBlocks = 3; };
template <int NF> struct LaunchTraits<cNutEqnAssemble<NF>> { static constexpr int minBlocks = 3; };
template <int NF> struct LaunchTraits<cPEqnAssemble<NF>> { static constexpr int minBlocks = 4; };
template <int NF> struct LaunchTraits<cPhiUpdate<NF>> { static constexpr int minBlocks = 4; };
// resident CTAs per SM of the compressible reverse kernels: cRevA 4, cRevB 3 (168 registers, with spills), cRevE (+cRevC) 4 --
// these kernels wait on gathers: more warps beat fewer spills
#ifndef DAB_CREVA_MINBLOCKS
#define DAB_CREVA_MINBLOCKS 4
#endif
#ifndef DAB_CREVB_MINBLOCKS
#define DAB_CREVB_MINBLOCKS 3
#endif
#ifndef DAB_CREVE_MINBLOCKS
#define DAB_CREVE_MINBLOCKS 4
#endif
template <int NF> struct LaunchTraits<cRevB<NF>> { static constexpr int minBlocks = DAB_CREVB_MINBLOCKS; };
template <int NF> struct LaunchTraits<cRevA<NF>> { static constexpr int minBlocks = DAB_CREVA_MINBLOCKS; };
template <int NF> struct LaunchTraits<cRevE<NF>> { static constexpr int minBlocks = DAB_CREVE_MINBLOCKS; };
template <int NF> struct LaunchTraits<cRevC<NF>> { static constexpr int minBlocks = 4; };
template <int NF> struct LaunchTraits<cFwdE<NF>> { static constexpr int minBlocks = 4; };
template <int NF> struct LaunchTraits<cFwdC<NF>> { static constexpr int minBlocks = 4; };
#endif

} // namespace dab
