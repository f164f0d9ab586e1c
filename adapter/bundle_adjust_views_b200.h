// bundle_adjust_views_b200.h -- BundleAdjustView (src/theia/sfm/bundle_adjustment/bundle_adjustment.cc:83-93) for many views
// in one engine call: what LocalizeViewToReconstruction (localize_view_to_reconstruction.cc:246-252) runs for every view a
// round of incremental / hybrid SfM localizes.  Gather the views' cameras, intrinsics groups and observations once, upload,
// tba_adjust_views, scatter the free coordinates back.  No CPU fallback.
#ifndef THEIA_SFM_BUNDLE_ADJUST_VIEWS_B200_H_
#define THEIA_SFM_BUNDLE_ADJUST_VIEWS_B200_H_

#include <vector>

#include "bundle_adjuster_b200.h"

namespace theia {

// The result of BundleAdjustView(options, view_ids[i], reconstruction) called for i = 0, 1, ... in that order: one summary per
// view.  Views whose intrinsics group has a free coordinate and was adjusted by an earlier view of the list see that view's
// intrinsics, as the sequential calls would; such views go into a later engine call on the same upload.  A view that is not
// estimated keeps its parameters and gets success = false, as does every view when no GPU is usable.
std::vector<BundleAdjustmentSummary> BundleAdjustViewsB200(const BundleAdjustmentOptions& options, const std::vector<ViewId>& view_ids,
                                                           Reconstruction* reconstruction);

}  // namespace theia
#endif
