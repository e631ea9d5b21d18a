// A DBoW2::FeatureVector (std::map<NodeId, std::vector<unsigned int>>) as the CSR the _fv entries of libcubemap_b200.so take: the map's nodes
// in map order (strictly ascending), fv_start with count + 1 offsets, the features of each node in list order. Shared by the drop-ins that
// pass mFeatVec to the device; a frame of n features fills a CSR of stride max(n, 1).
#pragma once
#include <cstdint>
#include <vector>

#include "ThirdParty/DBoW2/DBoW2/FeatureVector.h"

namespace cubemap_b200 {
struct FeatureVectorCsr {
    std::vector<int32_t> node, start, feat;
    int32_t count = 0;
    FeatureVectorCsr(const DBoW2::FeatureVector& fv, int stride) : node(stride, 0), start(stride + 1, 0), feat(stride, 0) {
        int32_t k = 0;
        for (DBoW2::FeatureVector::const_iterator it = fv.begin(); it != fv.end(); ++it, ++count) {
            node.at(count) = (int32_t)it->first;   // at(): a FeatureVector listing more than `stride` features throws instead of overrunning
            for (size_t i = 0; i < it->second.size(); i++) feat.at(k++) = (int32_t)it->second[i];
            start[count + 1] = k;
        }
    }
};
}  // namespace cubemap_b200
