// Stand-in for rtabmap::Memory as the reference's BayesFilter.cpp sees it.  TEST INFRASTRUCTURE ONLY.
//
// The graph walk of Memory::getNeighborsId is not what the oracle pins: the caller loads, for every place, the neighbour
// table {neighbour id: graph margin} the walk would return, and getNeighborsId hands it back limited to margins below
// maxGraphDepth.  isInSTM answers from a caller-loaded set of short-term-memory ids.
#pragma once
#include <map>
#include <set>

namespace rtabmap {

class Memory
{
public:
	std::map<int, int> getNeighborsId(int signatureId, int maxGraphDepth, int maxCheckedInDatabase = -1, bool incrementMarginOnLoop = false,
	                                  bool ignoreLoopIds = false, bool ignoreIntermediateNodes = false, bool ignoreLocalSpaceLoopIds = false,
	                                  const std::set<int> & nodesSet = std::set<int>(), double * dbAccessTime = 0) const
	{
		(void)maxCheckedInDatabase; (void)incrementMarginOnLoop; (void)ignoreLoopIds; (void)ignoreIntermediateNodes;
		(void)ignoreLocalSpaceLoopIds; (void)nodesSet; (void)dbAccessTime;
		std::map<int, int> out;
		const std::map<int, std::map<int, int> >::const_iterator it = neighbors.find(signatureId);
		if (it != neighbors.end())
			for (const auto & kv : it->second)
				if (kv.second < maxGraphDepth) out.insert(kv);
		return out;
	}
	bool isInSTM(int signatureId) const { return stm.find(signatureId) != stm.end(); }

	std::map<int, std::map<int, int> > neighbors; // loaded by the caller
	std::set<int> stm;
};

} // namespace rtabmap
