/*
 * GpuCacheMissLB — replaces ModelMesh.CacheMissForwardingLB (ModelMesh.java:4757-5005) at its factory call site
 * (ModelMesh.java:1107-1110: ThriftClientBuilder.withLoadBalancer(...)).  Same litelinks LoadBalancer SPI, same three results
 * (a ServiceInstanceInfo, null, LoadBalancer.ABORT_REQUEST), same side effects on the per-request CacheMissExcludeSet and
 * thread context (ModelMesh.java:4992-5003).  On any library error it delegates to the existing Java implementation -- the
 * library has no CPU path of its own.  Source only (litelinks is not vendored in the build image).
 */
package com.ibm.watson.modelmesh.gpu;

import java.util.Map;

import com.ibm.watson.litelinks.client.LoadBalancer;
import com.ibm.watson.litelinks.client.LoadBalancingPolicy.InclusiveLoadBalancingPolicy;

public abstract class GpuCacheMissLB implements LoadBalancer {
    /** What the LB needs from the enclosing ModelMesh instance (all exist there today as fields / methods). */
    public interface Host {
        String instanceId();
        String requestModelId();                                   // the model the current request is about
        String requestModelType();                                 // CacheMissExcludeSet.modelType: the record's type (MM:3782)
        java.util.Set<String> requestLoadedAndFailed();            // its loaded / failed key sets: the record read for this request
                                                                   // (MM:3537, 3785 -> 4735-4743; refreshed after a failed load MM:4088-4097)
        java.util.Set<String> requestExcludes();                   // CacheMissExcludeSet's own members ∪ explicit (MM:4706-4715)
        long requestLastUsedTime();                                // CacheMissExcludeSet.lastUsedTime (MM:4730)
        boolean requestFavourSelf();                               // CacheMissExcludeSet.favourSelf (MM:4721)
        com.ibm.watson.modelmesh.InstanceRecord freshInstanceRecord();  // getFreshInstanceRecord() (MM:5369)
        void requestExcludeAdd(String instanceId);                 // exclude.add(chosen) + context keys (MM:4992-5003)
        <T> T fallback(Object[] sis, String method, Object[] args); // the Java CacheMissForwardingLB
        <T> Map<String, T> serviceInstanceMap(Object[] sis);       // ForwardingLB.getMap (MM:4299-4313)
    }

    private final GpuPlacement gpu;
    private final Host host;

    protected GpuCacheMissLB(GpuPlacement gpu, Host host) { this.gpu = gpu; this.host = host; }

    @Override
    @SuppressWarnings("unchecked")
    public <T> T getNext(Object[] sis, String method, Object[] args) {
        final String chosen;
        try {
            chosen = gpu.placeOne(host.requestModelType(), host.requestLoadedAndFailed(), host.instanceId(), host.requestLastUsedTime(),
                    host.requestFavourSelf(), host.freshInstanceRecord(), host.requestExcludes(), System.currentTimeMillis());
        } catch (RuntimeException e) {  // library error
            return host.fallback(sis, method, args);
        }
        if (chosen == null) return null;                                      // MM:4796, 4941: "Nowhere available to load" upstream
        if (chosen == GpuPlacement.SELF) return (T) LoadBalancer.ABORT_REQUEST;  // MM:4894, 4990
        T si = (T) host.serviceInstanceMap(sis).get(chosen);
        if (si == null) return host.fallback(sis, method, args);              // the snapshot named an instance litelinks no longer lists
        host.requestExcludeAdd(chosen);
        return si;
    }
}
