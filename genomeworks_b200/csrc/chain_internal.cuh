// gw-b200: the chainer's call for engines that hand the chain's SSPs straight to the next stage (genome_aligner_capi.cu).
#pragma once

#include <cstdint>

#include "../../include/gwb200.h"

namespace gwb200
{
namespace chain
{

// gwb200_ssp_chainer_chain_device, which also writes the chain's SSPs to d_out (room for n records) in ascending index.
int chain_ssps(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty, void* d_out);
// gwb200_ssp_chainer_chain_all_device, which also writes the union's SSPs to d_out (room for n records) in ascending index.
int chain_all_ssps(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty, int64_t min_score,
                   void* d_out);

} // namespace chain
} // namespace gwb200
